"""GPU: weighted dense adjacency on every kernel that reads slot weights, against float64.

A weighted ``[b, T, v, v]`` matrix is scanned into per-type message lists, per-slot weights (``slot_w`` in target-CSR order, ``tslot_w``
in source-CSR order) and fp32 row sums; the forward kernels scale each message by its slot weight (the GLOBAL tile kernel's
4-rows-in-flight accumulate, the LOCAL tile kernels' gather without the shared-memory CSR cache, every fp32 instance, the per-timestep
fp32 path), the backward's two gathers by ``slot_w`` and ``tslot_w``, and the edge-bias term and its gradient use the row sums.  The
batches, regimes and cases are built in tests/test_weighted_dense_cpu.py, which asserts their shapes and pins their binary twins'
plans without a GPU.  Here every case asserts its own plan text on the device (ending in the weighted suffix) and compares with the
float64 dense oracle (``dense_propagation_loops``; ``dense_propagation_torch`` with the engine's mask under state dropout):

* forward: the final state, every bias drawn nonzero; bars max|err| / max|ref| of tests/test_gpu_forward_plans.py (fp32 1e-5, bf16x3
  1e-4, bf16 2e-2), per graph for the batch whose graphs' weights span 1e-3 to 1e3;
* the host scan at 1, 2, 3 and 8 threads: the same image bytes and forward bits, the last-graph-only matrix weighted at each;
* gradients: ``d h0`` and every weight and bias gradient (``edge_biases`` included) against float64 autograd with the state-dropout mask
  replayed, under both backward precisions; bars 2.5e-5 on an fp32 forward with the fp32 backward, else 2e-4;
* deterministic mode: every gradient the same bits across two calls and on a fresh engine.
"""
import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests.test_backward_plans_cpu import plan_matches
from tests.test_weighted_dense_cpu import (CASES, DETERMINISM, EDGE, FFMA, GRAD_CASES, HOST_THREADS, STEP, TILE, WEIGHTED_TAG, binary, case_h0,
                                           h0_for, weigh)

pytestmark = pytest.mark.gpu

BARS = {"fp32": 1e-5, "bf16x3": 1e-4, "bf16": 2e-2}
DROP_SEED = 20261017


def _set_env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _weights(c, T):
    """The dense initialisers with the zero candidate bias drawn: every bias (gate, candidate, edge) is nonzero."""
    dw = O.init_dense_weights({"hidden_size": c.D, "use_edge_bias": c.bias}, T, np.random.default_rng(5))
    dw["cand_bias"] = np.random.default_rng(6).normal(0, 0.1, c.D).astype(np.float32)
    return dw


def _engine_weights(dw, T, D):
    w = dict(dw)
    if "edge_biases" in w:
        w["edge_biases"] = w["edge_biases"].reshape(T, D)
    return [w]


def _engine(c, dw, T, A):
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(c.params, T, precision=c.precision)
    eng.set_weights(U.to_cuda_weights(_engine_weights(dw, T, c.D)))
    if c.keep < 1.0:
        eng.set_state_dropout(c.keep, DROP_SEED)
    eng.set_graph_dense(A)
    return eng


def _check_plan(c, plan):
    assert plan.endswith(WEIGHTED_TAG), (c.name, plan)
    assert plan_matches(plan, c.pattern), (c.name, c.pattern, plan)


def _reference(c, A, h0, dw):
    import torch
    p = {"num_timesteps": c.steps, "use_edge_bias": c.bias}
    if c.keep < 1.0:
        return O.dense_propagation_torch(h0, A, dw, p, dtype=torch.float64, state_dropout=(c.keep, DROP_SEED)).numpy()
    return O.dense_propagation_loops(h0, A, dw, p, dtype=np.float64)


def _forward(c, monkeypatch):
    import torch
    _set_env(monkeypatch, c.env)
    A = c.matrix()
    b, T, v, _ = A.shape
    h0 = case_h0(c, A)
    dw = _weights(c, T)
    eng = _engine(c, dw, T, A)
    _check_plan(c, eng.plan)
    out = eng.forward(torch.from_numpy(h0.reshape(b * v, c.D)).cuda())
    eng.sync_check()
    got = out.cpu().numpy().reshape(b, v, c.D)
    ref = _reference(c, A, h0, dw)
    bar = BARS[c.precision]
    if c.regime == "scales":   # per graph: the 1e-3 graphs are not hidden by the 1e3 ones
        errs = [U.max_rel_err(got[g], ref[g]) for g in range(b)]
        print("\nWDENSE %-44s %.3e  per graph %s" % (c.name, max(errs), " ".join("%.1e" % e for e in errs)))
        for g, e in enumerate(errs):
            assert e < bar, (c.name, "graph %d" % g, e, bar)
    else:
        err = U.max_rel_err(got, ref)
        print("\nWDENSE %-44s %.3e" % (c.name, err))
        assert err < bar, (c.name, err, bar)
    return eng


# ---------------------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("case", [c.name for c in TILE])
def test_tile_kernel(case, monkeypatch):
    """The tile-local wgmma kernel at every NH, bf16x3 and bf16: compact LOCAL, 128-row LOCAL, GLOBAL through a 200-node component,
    forced GLOBAL."""
    _forward(CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [c.name for c in FFMA])
def test_ffma_instances(case, monkeypatch):
    """All twelve fp32 instances (variant x nb1 x LOCAL / GLOBAL)."""
    _forward(CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [c.name for c in STEP])
def test_stepwise(case, monkeypatch):
    """The per-timestep fp32 path at hidden 260 and 512."""
    _forward(CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [c.name for c in EDGE])
def test_edge_cases(case, monkeypatch):
    """T = 1; 16 types with three present; no edge bias; 1 and 8 timesteps; state keep 0.8; b = 1; v = 1, 2, 3, 5 with entries only in
    the scan's tail columns; self-loops; negative weights and rows that cancel to 0; 1.0 among weighted entries; per-graph scales 1e-3 to
    1e3; a 0/1 matrix but for one entry in its last graph.  Hidden 36 and 100, fp32 and bf16x3, LOCAL and GLOBAL."""
    _forward(CASES[case], monkeypatch)


# ---------------------------------------------------------------------------------------------------------------- host scan
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_host_scan_is_the_same_at_every_thread_count(precision, monkeypatch):
    """64 graphs scanned by 1, 2, 3 and 8 host threads: the same graph image bytes and the same forward bits; the matrix that is 0/1
    but for one entry in its last graph is weighted at every count (and matches the oracle)."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    from tests.test_weighted_dense_cpu import Case
    c = Case("scan", "mol64", "uniform", precision, 36, {}, r"^(fp32-ffma|wgmma-bf16x3) LOCAL\(")
    Abin = binary("mol64")
    b, T, v, _ = Abin.shape
    h0 = h0_for(Abin, c.D)
    dw = _weights(c, T)
    th0 = torch.from_numpy(h0.reshape(b * v, c.D)).cuda()
    runs = {}
    for regime in ("uniform", "lastonly"):
        A = weigh(Abin, regime)
        ref = _reference(c, A, h0, dw)
        for n in HOST_THREADS:
            monkeypatch.setenv("GGNN_HOST_THREADS", str(n))
            eng = PropagationEngine(c.params, T, precision=precision)
            eng.set_weights(U.to_cuda_weights(_engine_weights(dw, T, c.D)))
            eng.set_graph_dense(A)
            _check_plan(c, eng.plan)
            out = eng.forward(th0).cpu().numpy()
            eng.sync_check()
            runs.setdefault(regime, []).append((n, eng.graph_image(), out))
            err = U.max_rel_err(out.reshape(b, v, c.D), ref)
            print("\nWDENSE scan-%s-%s-threads%d %.3e" % (precision, regime, n, err))
            assert err < BARS[precision], (regime, n, err)
    for regime, rs in runs.items():
        for n, image, out in rs[1:]:
            np.testing.assert_array_equal(image, rs[0][1], err_msg="%s image at %d threads" % (regime, n))
            np.testing.assert_array_equal(out, rs[0][2], err_msg="%s forward at %d threads" % (regime, n))


# ---------------------------------------------------------------------------------------------------------------- gradients
def _autograd(c, A, h0, dw, g_out):
    import torch
    tw = {k: torch.tensor(x, dtype=torch.float64, requires_grad=True) for k, x in dw.items()}
    th0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    out = O.dense_propagation_torch(th0, A, tw, {"num_timesteps": c.steps, "use_edge_bias": c.bias}, dtype=torch.float64,
                                    state_dropout=(c.keep, DROP_SEED) if c.keep < 1.0 else None)
    (out * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
    return out.detach().numpy(), th0.grad.numpy(), {k: t.grad.numpy() for k, t in tw.items()}


class _Trained:
    """An engine after a forward with save_for_backward; ``backward()`` returns (d h0, {weight: gradient}) as NumPy."""

    def __init__(self, c, bwd, det=False):
        import torch
        self.c = c
        self.A = c.matrix()
        b, self.T, v, _ = self.A.shape
        self.h0 = case_h0(c, self.A)
        self.dw = _weights(c, self.T)
        self.g_out = np.random.default_rng(7).normal(size=self.h0.shape).astype(np.float32)
        from gated_graph_neural_network_samples_b200.engine import PropagationEngine
        self.eng = PropagationEngine(c.params, self.T, precision=c.precision)
        self.dev_w = U.to_cuda_weights(_engine_weights(self.dw, self.T, c.D))
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(True)
        self.eng.set_deterministic(det)
        self.eng.set_backward_precision(bwd)
        if c.keep < 1.0:
            self.eng.set_state_dropout(c.keep, DROP_SEED)
        self.eng.set_graph_dense(self.A)
        _check_plan(c, self.eng.plan)
        self.th0 = torch.from_numpy(self.h0.reshape(b * v, c.D)).cuda()
        self.out = self.eng.forward(self.th0)
        self.eng.sync_check()

    def backward(self):
        import torch
        grads = [{k: torch.zeros_like(t) for k, t in self.dev_w[0].items()}]
        dh0 = torch.zeros_like(self.th0)
        self.eng.backward(torch.from_numpy(self.g_out.reshape(self.th0.shape)).cuda(), grads, dh0)
        self.eng.sync_check()
        return dh0.cpu().numpy(), {k: t.cpu().numpy() for k, t in grads[0].items()}


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("case", sorted(GRAD_CASES))
def test_gradients_match_float64_autograd(case, bwd, monkeypatch):
    """tc compact, 128-row and GLOBAL (bf16x3 forward), fp32 variant 0 and 1 LOCAL, fp32 GLOBAL and stepwise at 260, plus the signed /
    cancelling regime on fp32 LOCAL and tc GLOBAL; state keep 0.8 with the engine's mask replayed; both backward precisions."""
    c = GRAD_CASES[case]
    _set_env(monkeypatch, c.env)
    t = _Trained(c, bwd)
    dh0, gw = t.backward()
    out, rdh0, rgw = _autograd(c, t.A, t.h0, t.dw, t.g_out)
    b, v = t.h0.shape[:2]
    pairs = [("forward", t.out.cpu().numpy().reshape(b, v, c.D), out), ("d h0", dh0.reshape(b, v, c.D), rdh0)]
    pairs += [("d " + k, gw[k].reshape(rgw[k].shape), rgw[k]) for k in sorted(rgw)]
    assert sorted(gw) == sorted(rgw) and "edge_biases" in gw
    bar = 2.5e-5 if (c.precision, bwd) == ("fp32", "fp32") else 2e-4
    errs = [(U.max_rel_err(g, r), n) for n, g, r in pairs]
    print("\nWDENSEGRAD %-36s bwd %-6s forward %.2e  worst gradient %.2e on %s" % (case, bwd, errs[0][0], *max(errs[1:])))
    assert errs[0][0] < BARS[c.precision], (case, errs[0])
    for e, n in errs[1:]:
        assert e < bar, (case, bwd, n, e, bar)


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("case", DETERMINISM)
def test_deterministic_gradients_repeat(case, bwd, monkeypatch):
    """Under ggnn_set_deterministic: the forward and every gradient the same bits on two backward calls and on a fresh engine."""
    c = GRAD_CASES[case]
    _set_env(monkeypatch, c.env)
    a = _Trained(c, bwd, det=True)
    dh0, g1 = a.backward()
    dh0_2, g2 = a.backward()
    fresh = _Trained(c, bwd, det=True)
    dh0_3, g3 = fresh.backward()
    np.testing.assert_array_equal(a.out.cpu().numpy(), fresh.out.cpu().numpy())
    for other_dh0, other in ((dh0_2, g2), (dh0_3, g3)):
        np.testing.assert_array_equal(other_dh0, dh0)
        for k in g1:
            np.testing.assert_array_equal(other[k], g1[k], err_msg=k)
