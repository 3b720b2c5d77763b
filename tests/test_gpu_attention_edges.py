"""GPU: propagation attention at the edges of its kernels, forward and every gradient against float64.

The batches, score regimes and cases are tests/test_attention_edges_cpu.py's, which pins every case to its plan without a GPU.  Each
case runs a forward with save_for_backward and ``ggnn_backward``, and compares the forward with float64 and ``d h0`` and every weight
gradient of every layer (edge weights and biases, gate / candidate kernels and biases, ``cand_hidden_bias``,
``edge_type_attention_weights``) with float64 autograd of ``oracle.sparse_propagation_torch``; state dropout is replayed with the same
seed.  Bars, max|err| / max|ref| per tensor: forward 1e-5, gradients 2.5e-5; the large / negative score regimes and the 100 k-node batch
1e-4 (an fp32 score carries an error of about |score| 2^-24, and ``d a_t`` there is a sum of many thousand atomics).  The worst error of
each group is printed at the end (``-s``).

Groups: every accepted hidden size 4..256 on the default plan (the forward's second lane pass over the score dot product above hidden 128,
the target backward's column slots 4-7), and six of them on the 64-row tile variant and GLOBAL; in-degrees 1..65, 300 and 1100, self-
loops and duplicate messages, 16 edge types (all present / only 0 and 15: absent types must get a ``d a_t`` of exactly 0) and one, LOCAL
and GLOBAL; scores >= 90 and <= -90 at step 0, a_t = 0 and a_t < 0; attention with state dropout, CudnnCompatibleGRUCell, RNN, a
zero-step layer read through a residual and four residual inputs; partial gradient requests, accumulation into prefilled buffers,
bit-identical forward and ``d h0``; a batch of the reference's default size; the SparseGGNNChemModel plug-in in training.
"""
import time

import numpy as np
import pytest

from tests.test_attention_edges_cpu import (ABI_CASES, ATT_LOCAL, CASES, DEFAULT_SIZE_PARAMS, batch, default_size_batch, plan_matches,
                                            regime_h0, regime_weights)
from tests.test_gpu_backward import _autograd_reference, _engine_grads

pytestmark = pytest.mark.gpu

BAR_FORWARD, BAR_GRADIENT, BAR_WIDE = 1e-5, 2.5e-5, 1e-4
REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}
DROPOUT_SEED = 4321
WORST = {}   # group -> {"forward": (err, case), "gradient": (err, case, tensor)}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\n\nworst max|err|/max|ref| per group:")
        for g, w in WORST.items():
            print("  %-26s forward %.2e (%s)   gradient %.2e (%s, %s)" % (g, w["forward"][0], w["forward"][1], w["gradient"][0],
                                                                           w["gradient"][1], w["gradient"][2]))


def _set_env(monkeypatch, env):
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_FFMA_VARIANT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _rel(got, ref):
    ref = np.asarray(ref, np.float64)
    if not np.any(ref):
        return float(np.max(np.abs(got))) if got.size else 0.0
    return float(np.max(np.abs(got - ref)) / np.max(np.abs(ref)))


def _compare(group, name, got, ref, bar_forward, bar_gradient):
    (out, dh0, gw), (rout, rdh0, rgw) = got, ref
    assert np.all(np.isfinite(out)) and np.all(np.isfinite(dh0)), name
    pairs = [("d h0", dh0, rdh0)] + [("layer %d %s" % (l, k), a[k], r[k]) for l, (a, r) in enumerate(zip(gw, rgw)) for k in sorted(r)]
    assert any("edge_type_attention_weights" in n for n, _, _ in pairs)
    f_err = _rel(out, rout)
    errs = [(_rel(g, r), n) for n, g, r in pairs]
    worst = max(errs)
    print("\n%-28s forward %.2e  worst gradient %.2e on %s" % (name, f_err, worst[0], worst[1]))
    w = WORST.setdefault(group, {"forward": (0.0, ""), "gradient": (0.0, "", "")})
    w["forward"] = max(w["forward"], (f_err, name))
    w["gradient"] = max(w["gradient"], (worst[0], name, worst[1]))
    assert f_err < bar_forward, (name, "forward", f_err)
    bad = [(n, e) for e, n in errs if not e < bar_gradient]
    assert not bad, (name, bad)


def _inputs(c):
    adj, indeg, T = batch(c.kind)
    h0 = regime_h0(c.regime, indeg.shape[0], c.D)
    w = regime_weights(c.params, T, c.regime)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    return adj, indeg, T, h0, w, g_out


def _check_case(c, monkeypatch):
    _set_env(monkeypatch, c.env)
    adj, indeg, T, h0, w, g_out = _inputs(c)
    drop = (c.state_keep, DROPOUT_SEED) if c.state_keep < 1.0 else None
    ref = _autograd_reference(c.params, T, w, adj, indeg, h0, g_out, state_dropout=drop)
    plan = []

    def set_graph(e):
        e.set_graph_sparse(adj, indeg)
        plan.append(e.plan)

    got = _engine_grads(c.params, T, w, set_graph, h0, g_out, "fp32", state_dropout=drop)
    assert plan_matches(plan[0], c.plan), (c.plan, plan[0])
    wide = c.regime in ("large", "negative")
    _compare(c.group, c.name, got, ref, BAR_WIDE if wide else BAR_FORWARD, BAR_WIDE if wide else BAR_GRADIENT)
    return adj, got


@pytest.mark.parametrize("case", [n for n, c in CASES.items() if c.group == "hidden sweep"])
def test_hidden_sweep(case, monkeypatch):
    _check_case(CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [n for n, c in CASES.items() if c.group == "degree and topology"])
def test_degree_and_topology(case, monkeypatch):
    adj, (_, _, gw) = _check_case(CASES[case], monkeypatch)
    absent = [t for t, a in enumerate(adj) if a.shape[0] == 0]
    for lw in gw:
        assert np.all(lw["edge_type_attention_weights"][absent] == 0.0), lw["edge_type_attention_weights"]
        assert np.all(lw["edge_weights"][absent] == 0.0)
        assert np.all(lw["edge_type_attention_weights"][[t for t in range(len(adj)) if t not in absent]] != 0.0)


@pytest.mark.parametrize("case", [n for n, c in CASES.items() if c.group in ("large / negative scores", "a_t = 0 / a_t < 0")])
def test_score_regimes(case, monkeypatch):
    _check_case(CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [n for n, c in CASES.items() if c.group == "feature crosses"])
def test_feature_crosses(case, monkeypatch):
    _check_case(CASES[case], monkeypatch)


# ---------------------------------------------------------------------------------------------------------------- ABI behaviour
class _Trained:
    """One engine after a forward with save_for_backward on a case's batch; ``backward(fields)`` runs ggnn_backward into fresh zeroed
    buffers (or ``into``) for the requested weight fields of every layer."""

    def __init__(self, c, monkeypatch):
        import torch
        from gated_graph_neural_network_samples_b200.engine import PropagationEngine
        _set_env(monkeypatch, c.env)
        adj, indeg, T, h0, w, g_out = _inputs(c)
        self.eng = PropagationEngine(c.params, T, precision="fp32")
        self.dev_w = [{REN.get(k, k): torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda() for k, v in lw.items()} for lw in w]
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(True)
        self.eng.set_graph_sparse(adj, indeg)
        assert plan_matches(self.eng.plan, c.plan), (c.plan, self.eng.plan)
        self.h0 = torch.from_numpy(h0).cuda()
        self.g_out = torch.from_numpy(g_out).cuda()

    def forward(self):
        out = self.eng.forward(self.h0)
        self.eng.sync_check()
        return out.cpu().numpy()

    def fields(self):
        return sorted(self.dev_w[0])

    def zeros(self, fields):
        import torch
        return [{k: torch.zeros_like(lw[k]) for k in fields if k in lw} for lw in self.dev_w]

    def backward(self, fields, into=None):
        import torch
        grads = self.zeros(fields) if into is None else into
        dh0 = torch.zeros_like(self.h0)
        self.eng.backward(self.g_out, grads, dh0)
        self.eng.sync_check()
        return dh0.cpu().numpy(), [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]


NOISE = 1e-5   # the order noise of the atomics in the weight gradients (d a_t among them), relative to the largest entry


@pytest.mark.parametrize("case", ABI_CASES)
def test_partial_requests_and_prefilled_buffers(case, monkeypatch):
    """Only ``edge_type_attention_weights`` requested, and everything except it, against a full request (``d h0`` bit-identical); every
    gradient added into buffers prefilled with random values ends as prefill + gradient."""
    import torch
    t = _Trained(CASES[case], monkeypatch)
    t.forward()
    full_dh0, full = t.backward(t.fields())
    att = ["edge_type_attention_weights"]
    for request in (att, [k for k in t.fields() if k not in att]):
        dh0, part = t.backward(request)
        np.testing.assert_array_equal(dh0, full_dh0)
        for l, (p, f) in enumerate(zip(part, full)):
            assert sorted(p) == sorted(request)
            for k in p:
                assert _rel(p[k], f[k]) < NOISE, (l, k)
    rng = np.random.default_rng(9)
    pre = [{k: (rng.normal(size=v.shape) * np.max(np.abs(v))).astype(np.float32) for k, v in lw.items()} for lw in full]
    bufs = [{k: torch.from_numpy(v.copy()).cuda() for k, v in lw.items()} for lw in pre]
    dh0, acc = t.backward(t.fields(), into=bufs)
    np.testing.assert_array_equal(dh0, full_dh0)
    for l, (a, p, f) in enumerate(zip(acc, pre, full)):
        for k in a:
            assert np.max(np.abs(a[k] - (p[k].astype(np.float64) + f[k]))) <= NOISE * np.max(np.abs(f[k])), (l, k)


@pytest.mark.parametrize("case", ABI_CASES)
def test_forward_and_d_h0_are_bit_identical_run_to_run(case, monkeypatch):
    t = _Trained(CASES[case], monkeypatch)
    out_a = t.forward()
    dh0_a, _ = t.backward(t.fields())
    out_b = t.forward()
    dh0_b, _ = t.backward(t.fields())
    np.testing.assert_array_equal(out_a, out_b)
    np.testing.assert_array_equal(dh0_a, dh0_b)


# ---------------------------------------------------------------------------------------------------------------- default-size batch
def test_default_size_batch(monkeypatch):
    """About 100 k nodes (synthetic molecules and the hubs batch after them) at hidden 100: thousands of blocks add their ``d a_t`` with
    atomics.  Float64 autograd of it takes seconds on the CPU; the time is printed."""
    _set_env(monkeypatch, {})
    p = DEFAULT_SIZE_PARAMS
    adj, indeg = default_size_batch()
    V, D, T = indeg.shape[0], p["hidden_size"], 4
    h0 = regime_h0("mild", V, D)
    w = regime_weights(p, T, "mild")
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    t0 = time.perf_counter()
    ref = _autograd_reference(p, T, w, adj, indeg, h0, g_out)
    t_ref = time.perf_counter() - t0
    plan = []

    def set_graph(e):
        e.set_graph_sparse(adj, indeg)
        plan.append(e.plan)

    got = _engine_grads(p, T, w, set_graph, h0, g_out, "fp32")
    print("\ndefault-size batch: V=%d, %d messages, float64 autograd %.1f s, plan %s" % (V, sum(a.shape[0] for a in adj), t_ref, plan[0][:40]))
    assert plan_matches(plan[0], ATT_LOCAL), plan[0]
    _compare("default-size batch", "default-size-D100", got, ref, BAR_WIDE, BAR_WIDE)


# ---------------------------------------------------------------------------------------------------------------- through the plug-in
@pytest.mark.parametrize("hidden", [30, 100])
def test_plugin_training_batch_with_attention(tmp_path, monkeypatch, hidden):
    """SparseGGNNChemModel with attention: edge-weight keep 0.8, state keep 0.9, out-layer keep 0.9, two tasks with missing labels; the
    plug-in's own draws replayed (hidden 30 runs zero-padded to 32, its state-dropout mask drawn at the padded width)."""
    from tests.test_gpu_chem_ggnn_gradients import SPARSE_TRAINING, _check, _sparse_model, _training_feed, _two_task_molecules
    _set_env(monkeypatch, {})
    m = _sparse_model(tmp_path, "fp32", _two_task_molecules(64, seed=1), **dict(SPARSE_TRAINING, hidden_size=hidden,
                                                                                   use_propagation_attention=True))
    assert (m._padded_hidden != hidden) == (hidden % 4 != 0)
    _check("plug-in attention hidden %d" % hidden, m, _training_feed(m), monkeypatch, r"^fp32-ffma\+attention", "fp32")
