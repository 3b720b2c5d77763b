"""GPU: weighted dense adjacency on the streaming wgmma kernels (hidden sizes above 128 on bf16x3 / bf16), against float64.

The gather launch of a weighted batch sums every weighted (target, type) pair into a virtual row, ``sum_m w_m * (hi + lo)`` of its sources
in CSR order, and copies it like any other row; the pairs of one message of weight exactly 1 are copied from the source row itself.  The
batches, the tables' restatement and the plans at 132 SMs are checked without a GPU in tests/test_weighted_stream_cpu.py, which also
holds the float64 oracle used here (``weighted_propagation_torch``) to the dense and the sparse oracles.  Every case asserts its plan text
on the device (STREAM, weighted suffix).

* forward: the final state and every ``node_states_per_layer`` entry, bars max|err| / max|ref| 1e-4 (bf16x3) and 2e-2 (bf16); every
  K-step count per ring stage (``GGNN_TS_KSTEPS``) at hidden 132, 144, 192, 256, 260, 384 and 512 on both precisions; GRU and RNN/ReLU
  with and without edge bias, a residual input and state keep 0.8; the weight regimes (uniform, signed with zero row sums, 1.0 among
  weights, per-graph scales 1e-3 .. 1e3 at one timestep, one weighted entry in the last graph); hub rows of 12 messages in every batch;
* gradients: ``d h0`` and every weight and bias gradient against float64 autograd under both backward precisions, bar 2e-4;
* deterministic mode: the same forward and gradient bits across calls and on a fresh engine;
* one engine alternating weighted and binary streaming batches of different sizes: each result equal to a fresh engine's;
* the dense model at hidden 256: a 0/1 matrix streams through both dense entries with the same bits; a weighted one is refused by
  ``set_graph_dense`` and streams through ``set_graph_dense_weighted``; on fp32 both entries take it;
* canaries (tests/test_gpu_canaries.py's helpers): NaN graphs do not reach clean ones, forward and backward; guard bands around every
  caller buffer.
"""
import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests import test_canaries_cpu as K
from tests.test_backward_plans_cpu import plan_matches
from tests.test_gpu_backward import _cmp
from tests.test_gpu_canaries import REN, Ggnn, _g, _isolation
from tests.test_weighted_dense_cpu import BINARY_TAG, WEIGHTED_TAG
from tests.test_weighted_stream_cpu import STREAM_SIZES, TC_PRECISIONS, batch, matrix, params, stream_pattern, weighted_propagation_torch

pytestmark = pytest.mark.gpu

BARS = {"bf16x3": 1e-4, "bf16": 2e-2}
GRAD_BAR = 2e-4
DROP_SEED = 20261018


class Case:
    """One weighted streaming forward: batch, regime, precision, hidden size, model (cell, activation, edge bias, residual, state keep,
    timesteps) and GGNN_TS_KSTEPS (None: the engine's choice)."""

    def __init__(self, name, batch_name, regime, precision, D, cell="GRU", act="tanh", bias=True, residual=False, keep=1.0, steps=3, ks=None):
        self.name, self.batch, self.regime, self.precision, self.D = name, batch_name, regime, precision, D
        self.cell, self.act, self.bias, self.residual, self.keep, self.steps, self.ks = cell, act, bias, residual, keep, steps, ks

    @property
    def params(self):
        return params(self.D, self.steps, self.bias, self.cell, self.act, self.residual)

    def matrix(self):
        return matrix(self.batch, self.regime)


def _cases():
    out = []
    for D in STREAM_SIZES:                      # every K-step count at every hidden size, both precisions
        for prec in TC_PRECISIONS:
            for ks in (1, 2, 4):
                out.append(Case("ks%d-%s-D%d" % (ks, prec, D), "hub", "uniform", prec, D, ks=ks))
    for D in (256, 260):                        # the cells and model options
        for prec in TC_PRECISIONS:
            out += [Case("gru-nobias-%s-D%d" % (prec, D), "hub", "uniform", prec, D, bias=False),
                    Case("gru-residual-%s-D%d" % (prec, D), "hub", "uniform", prec, D, residual=True),
                    Case("gru-keep08-%s-D%d" % (prec, D), "hub", "uniform", prec, D, keep=0.8),
                    Case("rnn-relu-%s-D%d" % (prec, D), "hub", "uniform", prec, D, cell="RNN", act="relu"),
                    Case("rnn-relu-nobias-residual-%s-D%d" % (prec, D), "hub", "uniform", prec, D, cell="RNN", act="relu", bias=False,
                         residual=True),
                    Case("rnn-relu-keep08-%s-D%d" % (prec, D), "hub", "uniform", prec, D, cell="RNN", act="relu", keep=0.8)]
    for D in (256, 512):                        # the weight regimes
        for prec in TC_PRECISIONS:
            out += [Case("signed-%s-D%d" % (prec, D), "hub", "signed", prec, D),
                    Case("ones-%s-D%d" % (prec, D), "hub", "ones", prec, D),
                    Case("scales-%s-D%d" % (prec, D), "hub", "scales", prec, D, steps=1, bias=False),
                    Case("lastonly-%s-D%d" % (prec, D), "hub64", "lastonly", prec, D),
                    Case("big-components-%s-D%d" % (prec, D), "one200", "uniform", prec, D)]
    return out


CASES = {c.name: c for c in _cases()}
assert len(CASES) == len(_cases())


def _env(monkeypatch, c):
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM", "GGNN_TS_KSTEPS"):
        monkeypatch.delenv(k, raising=False)
    if c.ks:
        monkeypatch.setenv("GGNN_TS_KSTEPS", str(c.ks))


def _weights(c, T):
    """The sparse initialisers with every bias drawn nonzero; oracle names (rnn_kernel / rnn_bias for the RNN cell)."""
    w = O.init_sparse_weights(c.params, T, np.random.default_rng(5))
    rng = np.random.default_rng(6)
    for lw in w:
        for k in ("cand_bias", "rnn_bias"):
            if k in lw:
                lw[k] = rng.normal(0, 0.1, lw[k].shape).astype(np.float32)
    return w


def _h0(c, A):
    """h0 [b*v, D]; the ``scales`` regime divides each graph's states by its scale where it exceeds 1 (as tests/test_weighted_dense_cpu.py
    does), so that its messages stay O(1)."""
    b, _, v, _ = A.shape
    h0 = np.random.default_rng(500 + c.D).normal(0, 1, (b, v, c.D)).astype(np.float32)
    if c.regime == "scales":
        h0 = (h0 / np.maximum(np.logspace(-3, 3, b), 1.0)[:, None, None]).astype(np.float32)
    return h0.reshape(b * v, c.D)


def _drop(c):
    return (c.keep, DROP_SEED) if c.keep < 1.0 else None


def _engine(c, w, T, A, save=False, det=False, bwd=None):
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(c.params, T, precision=c.precision)
    dev_w = U.to_cuda_weights([{REN.get(k, k): x for k, x in lw.items()} for lw in w])
    eng.set_weights(dev_w)
    eng.set_save_for_backward(save)
    eng.set_deterministic(det)
    if bwd:
        eng.set_backward_precision(bwd)
    if c.keep < 1.0:
        eng.set_state_dropout(c.keep, DROP_SEED)
    eng.set_graph_dense_weighted(A)
    tag = WEIGHTED_TAG if np.any((A != 0) & (A != 1)) else BINARY_TAG
    assert eng.plan.endswith(tag) and plan_matches(eng.plan, stream_pattern(c.precision, c.D)), (c.name, eng.plan)
    return eng, dev_w


# ---------------------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("case", sorted(CASES))
def test_forward_matches_float64(case, monkeypatch):
    import torch
    c = CASES[case]
    _env(monkeypatch, c)
    A = c.matrix()
    b, T, v, _ = A.shape
    w = _weights(c, T)
    h0 = _h0(c, A)
    eng, _ = _engine(c, w, T, A, save=True)
    eng.forward(torch.from_numpy(h0).cuda())
    got = [eng.layer_state(l).cpu().numpy() for l in range(eng.L + 1)]
    eng.sync_check()
    ref = [r.numpy() for r in weighted_propagation_torch(h0, A, w, c.params, state_dropout=_drop(c), return_all_layers=True)]
    assert len(got) == len(ref)
    bar = BARS[c.precision]
    errs = []
    for l, (g, r) in enumerate(zip(got, ref)):
        if c.regime == "scales":   # per graph: the 1e-3 graphs are not hidden by the 1e3 ones
            errs.append(max(U.max_rel_err(g.reshape(b, v, -1)[i], r.reshape(b, v, -1)[i]) for i in range(b)))
        else:
            errs.append(U.max_rel_err(g, r))
    print("\nWSTREAM %-40s layers %s" % (case, " ".join("%.2e" % e for e in errs)))
    for l, e in enumerate(errs):
        assert e < bar, (case, "node_states_per_layer[%d]" % l, e, bar)


# ---------------------------------------------------------------------------------------------------------------- gradients
GRAD = [Case("grad-gru-keep08-D256", "hub", "uniform", "bf16x3", 256, keep=0.8),
        Case("grad-rnn-relu-residual-signed-D260", "hub", "signed", "bf16x3", 260, cell="RNN", act="relu", residual=True),
        Case("grad-gru-residual-ones-D512", "hub", "ones", "bf16x3", 512, residual=True),
        Case("grad-gru-nobias-D132", "hub", "uniform", "bf16x3", 132, bias=False)]
GRAD_CASES = {c.name: c for c in GRAD}


class _Trained:
    def __init__(self, c, bwd, det=False):
        import torch
        self.c = c
        self.A = c.matrix()
        self.T = self.A.shape[1]
        self.w = _weights(c, self.T)
        self.h0 = _h0(c, self.A)
        self.g_out = np.random.default_rng(7).normal(size=self.h0.shape).astype(np.float32)
        self.eng, self.dev_w = _engine(c, self.w, self.T, self.A, save=True, det=det, bwd=bwd)
        self.th0 = torch.from_numpy(self.h0).cuda()
        self.out_t = self.eng.forward(self.th0)   # kept alive: the backward reads node_states_per_layer[L] (the RNN cell's derivative)
        self.out = self.out_t.cpu().numpy()
        self.eng.sync_check()

    def backward(self):
        import torch
        grads = [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in self.dev_w]
        dh0 = torch.zeros_like(self.th0)
        self.eng.backward(torch.from_numpy(self.g_out).cuda(), grads, dh0)
        self.eng.sync_check()
        return dh0.cpu().numpy(), [{k: t.cpu().numpy() for k, t in lw.items()} for lw in grads]


def _autograd(c, A, h0, w, g_out):
    import torch
    tw = [{k: torch.tensor(x, dtype=torch.float64, requires_grad=True) for k, x in lw.items()} for lw in w]
    th0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    out = weighted_propagation_torch(th0, A, tw, c.params, state_dropout=_drop(c))
    (out * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
    return out.detach().numpy(), th0.grad.numpy(), [{REN.get(k, k): t.grad.numpy() for k, t in lw.items()} for lw in tw]


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("case", sorted(GRAD_CASES))
def test_gradients_match_float64_autograd(case, bwd, monkeypatch):
    c = GRAD_CASES[case]
    _env(monkeypatch, c)
    t = _Trained(c, bwd)
    dh0, gw = t.backward()
    out, rdh0, rgw = _autograd(c, t.A, t.h0, t.w, t.g_out)
    pairs = [("d h0", dh0, rdh0)]
    for l, (g, r) in enumerate(zip(gw, rgw)):
        assert sorted(g) == sorted(r), (sorted(g), sorted(r))
        pairs += [("layer %d d %s" % (l, k), g[k].reshape(r[k].shape), r[k]) for k in sorted(r)]
    fwd = U.max_rel_err(t.out, out)
    errs = [(U.max_rel_err(g, r), n) for n, g, r in pairs]
    print("\nWSTREAMGRAD %-36s bwd %-6s forward %.2e  worst gradient %.2e on %s" % (case, bwd, fwd, *max(errs)))
    assert fwd < BARS[c.precision], (case, fwd)
    for e, n in errs:
        assert e < GRAD_BAR, (case, bwd, n, e)


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("case", ["grad-gru-keep08-D256", "grad-gru-residual-ones-D512"])
def test_deterministic_forward_and_gradients_repeat(case, bwd, monkeypatch):
    c = GRAD_CASES[case]
    _env(monkeypatch, c)
    a = _Trained(c, bwd, det=True)
    dh0, g1 = a.backward()
    dh0_2, g2 = a.backward()
    fresh = _Trained(c, bwd, det=True)
    dh0_3, g3 = fresh.backward()
    np.testing.assert_array_equal(a.out, fresh.out)
    for other_dh0, other in ((dh0_2, g2), (dh0_3, g3)):
        np.testing.assert_array_equal(other_dh0, dh0)
        for l, lw in enumerate(g1):
            for k in lw:
                np.testing.assert_array_equal(other[l][k], lw[k], err_msg="layer %d %s" % (l, k))


# ---------------------------------------------------------------------------------------------------------------- one engine, many batches
def test_one_engine_alternates_weighted_and_binary_batches(monkeypatch):
    """Weighted molecules with hubs, their 0/1 twin, 64 weighted molecules (more virtual rows), one weighted molecule (fewer), two
    200-node components, then the first batch again: every forward and gradient equal to a fresh engine's on that batch."""
    import torch
    c = Case("mix", "hub", "uniform", "bf16x3", 256)
    _env(monkeypatch, c)
    seq = [matrix("hub", "uniform"), batch("hub"), matrix("hub64", "signed"), matrix("mol", "ones")[:1], matrix("one200", "uniform"),
           matrix("hub", "uniform")]
    T = seq[0].shape[1]
    w = _weights(c, T)
    eng = None

    def run(e, A, dev_w):
        e.set_graph_dense_weighted(A)
        want = WEIGHTED_TAG if np.any((A != 0) & (A != 1)) else BINARY_TAG
        assert e.plan.endswith(want) and plan_matches(e.plan, stream_pattern("bf16x3", 256)), e.plan
        h0 = torch.from_numpy(_h0(c, A)).cuda()
        out_t = e.forward(h0)   # kept alive until the backward has run
        out = out_t.cpu().numpy()
        grads = [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in dev_w]
        dh0 = torch.zeros_like(h0)
        e.backward(torch.from_numpy(np.random.default_rng(3).normal(size=h0.shape).astype(np.float32)).cuda(), grads, dh0)
        e.sync_check()
        return [out, dh0.cpu().numpy()] + [t.cpu().numpy() for lw in grads for t in lw.values()]

    for i, A in enumerate(seq):
        if eng is None:
            eng, dev_w = _engine(c, w, T, A, save=True, det=True)
        fresh, fresh_w = _engine(c, w, T, A, save=True, det=True)
        for a, b in zip(run(eng, A, dev_w), run(fresh, A, fresh_w)):
            np.testing.assert_array_equal(a, b, err_msg="batch %d" % i)


# ---------------------------------------------------------------------------------------------------------------- canaries
class _WeightedGgnn(Ggnn):
    """tests/test_gpu_canaries.py's runner, its dense matrix fed through set_graph_dense_weighted."""

    def set_graph(self, graph):
        self.eng.set_graph_dense_weighted(graph)


@pytest.mark.parametrize("D", [256, 512])
def test_poisoned_graphs_do_not_reach_clean_ones(D, monkeypatch):
    """Payload-NaN h0 and d_out in whole graphs (tests/test_gpu_canaries.py's rule): the clean graphs' states and d h0 keep their bits;
    with those graphs at 100x and d_out 0, the weight gradients repeat and match float64 autograd."""
    import torch
    c = Case("iso", "hub64", "uniform", "bf16x3", D)
    _env(monkeypatch, c)
    A = c.matrix()
    b, T, v, _ = A.shape
    w = _weights(c, T)
    r = _WeightedGgnn(c.params, T, w, "bf16x3", A)
    assert r.eng.plan.endswith(WEIGHTED_TAG) and plan_matches(r.eng.plan, stream_pattern("bf16x3", D)), r.eng.plan

    def ref(h, g):
        tw = [{k: torch.tensor(x, dtype=torch.float64, requires_grad=True) for k, x in lw.items()} for lw in w]
        th = torch.tensor(h, dtype=torch.float64, requires_grad=True)
        out = weighted_propagation_torch(th, A, tw, c.params)
        (out * torch.tensor(g, dtype=torch.float64)).sum().backward()
        return out.detach().numpy(), th.grad.numpy(), [{REN.get(k, k): t.grad.numpy() for k, t in lw.items()} for lw in tw]

    h0 = _h0(c, A)
    g = np.random.default_rng(7).normal(size=h0.shape).astype(np.float32)
    bad = np.repeat(np.isin(np.arange(b), K.poisoned_components(b)), v)
    _isolation("weighted stream D%d" % D, r, bad, h0, g, ref, _cmp)


@pytest.mark.parametrize("D", [132, 260, 512])
def test_guard_bands_around_every_buffer(D, monkeypatch):
    """Forward with save and backward with every caller pointer guarded (h0, h_out, every weight, d_out, d h0, every gradient prefilled),
    against the same calls on plain buffers: the same bits, no payload word in an output, every band intact."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    c = Case("guard", "hub", "signed", "bf16x3", D, residual=True)
    _env(monkeypatch, c)
    A = c.matrix()[:3, :, :17]   # 3 graphs of 17 rows: the last streaming tile ends at row 51
    A = np.ascontiguousarray(A[:, :, :, :17])
    b, T, v, _ = A.shape
    V = b * v
    w = _weights(c, T)
    rng = np.random.default_rng(9)
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    g = rng.normal(0, 1, (V, D)).astype(np.float32)
    pre = [{REN.get(k, k): rng.normal(0, 1, x.shape).astype(np.float32) for k, x in lw.items()} for lw in w]

    def run(guard):
        eng = PropagationEngine(c.params, T, precision="bf16x3")
        eng.set_deterministic(True)
        keep = []

        def buf(s, f=None):
            if guard:
                gb = _g(s, f)
                keep.append(gb)
                return gb.t
            return (torch.from_numpy(np.ascontiguousarray(f, np.float32)).cuda() if f is not None else torch.empty(s, device="cuda")).reshape(s)
        dev_w = [{REN.get(k, k): buf(x.shape, x) for k, x in lw.items()} for lw in w]
        eng.set_weights(dev_w)
        eng.set_save_for_backward(True)
        eng.set_graph_dense_weighted(A)
        assert eng.plan.endswith(WEIGHTED_TAG) and plan_matches(eng.plan, stream_pattern("bf16x3", D)), eng.plan
        th0, out = buf((V, D), h0), buf((V, D))
        eng.forward(th0, out)
        grads = [{k: buf(x.shape, x) for k, x in lw.items()} for lw in pre]
        dh0 = buf((V, D))
        eng.backward(buf((V, D), g), grads, dh0)
        eng.sync_check()
        outs = [out, dh0] + [t for lw in grads for t in lw.values()]
        if guard:
            assert not any(K.has_payload(t) for t in outs)
            assert all(gb.bands_intact() for gb in keep)
        return [t.cpu().numpy() for t in outs]

    for a, b_ in zip(run(True), run(False)):
        np.testing.assert_array_equal(a, b_)


def test_dense_entries_at_hidden_256():
    """The dense model at hidden 256 on 20 molecules in bucket 32.  A 0/1 matrix streams on bf16x3 through both entries with the same
    bits; the same matrix at 0.5 is refused by set_graph_dense there (as it always was) and streams through set_graph_dense_weighted;
    every run that is taken matches the float64 dense oracle at 1e-4, fp32 included."""
    import torch
    from gated_graph_neural_network_samples_b200 import packing, synthetic
    from gated_graph_neural_network_samples_b200.engine import GgnnError, PropagationEngine
    D, T, steps = 256, 4, 2
    mols = synthetic.make_molecules(20, seed=9)
    db = packing.pack_dense_batch(mols, 32, D, T)
    h0 = (db["initial_node_representation"] + np.random.default_rng(2).normal(0, 0.1, db["initial_node_representation"].shape)).astype(np.float32)
    dw = O.init_dense_weights({"hidden_size": D}, T, np.random.default_rng(5))
    dp = {"num_timesteps": steps, "use_edge_bias": True}
    binary = np.asarray(db["adjacency_matrix"], np.float32)

    def run(A, precision, entry):
        eng = PropagationEngine(U.dense_params_as_engine_params(dp, D), T, precision=precision)
        eng.set_weights(U.to_cuda_weights([dict(dw, edge_biases=np.asarray(dw["edge_biases"]).reshape(T, D))]))
        getattr(eng, entry)(A)
        got = eng.forward(torch.from_numpy(h0.reshape(-1, D)).cuda()).cpu().numpy().reshape(h0.shape)
        eng.sync_check()
        err = U.max_rel_err(got, O.dense_propagation_loops(h0, A, dw, dp))
        print("\nWSTREAM dense-D256 %s %s %s %.2e" % (entry, precision, eng.plan.rsplit("[", 1)[-1], err))
        assert err < 1e-4, (entry, precision, err)
        return eng.plan, got

    pb, gb = run(binary, "bf16x3", "set_graph_dense")
    pw, gw = run(binary, "bf16x3", "set_graph_dense_weighted")
    assert pb == pw and "STREAM" in pb and pb.endswith(BINARY_TAG), (pb, pw)
    np.testing.assert_array_equal(gb, gw)
    with pytest.raises(GgnnError, match="ggnn_set_graph_dense_weighted"):
        run(binary * 0.5, "bf16x3", "set_graph_dense")
    plan, _ = run(binary * 0.5, "bf16x3", "set_graph_dense_weighted")
    assert plan.endswith(WEIGHTED_TAG) and plan_matches(plan, stream_pattern("bf16x3", D)), plan
    for entry in ("set_graph_dense", "set_graph_dense_weighted"):
        plan, _ = run(binary * 0.5, "fp32", entry)
        assert plan.endswith(WEIGHTED_TAG) and "STREAM" not in plan, plan
