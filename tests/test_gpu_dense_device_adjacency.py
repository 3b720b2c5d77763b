"""GPU: the dense model's adjacency as a device tensor (ggnn_prepare_graph_dense_device, DESIGN §2.14) against float64.

A batch prepared from (b, v) alone takes its ``[b, T, v, v]`` matrix on the device (``set_message_weights``); ``backward(...,
d_message_weights=dA)`` adds the matrix's gradient at every entry.  Bars, max|err| / max|ref|: forward 1e-5 (fp32), 1e-4 (bf16x3), 2e-2
(bf16), as in tests/test_gpu_weighted_dense.py; gradients 2.5e-5 for an fp32 forward with the fp32 backward, else 2e-4.  Covered here:

* forward at hidden 4, 100, 128, 132, 256 and 512 on every precision, T = 1, 4 and 32, v = 1, 29, 128 and 300; 0/1, full soft, negative,
  all-zero matrices and per-graph scales from 1e-3 to 1e3 (checked per graph); state dropout, edge bias on and off, a multi-layer RNN with a
  residual, and b = 0;
* gradients of d h0, every weight and bias and dA against float64 autograd (dropout mask replayed) at both backward precisions;
* bit-repeatability of every gradient on two calls and on a fresh engine, in both deterministic modes;
* fp32 at hidden 260 and 512 on a 0/1 matrix: the forward and every gradient bit-identical to ``set_graph_dense``;
* the lifecycle (a forward before the matrix, a re-set before the backward, a new matrix on one prepared batch);
* memory canaries: NaN graphs beside clean ones, guard bands around the matrix, its gradient and every state buffer;
* the plug-in: two DenseGGNNChemModel training steps on a learnable per-type scale of the adjacency, its gradient against float64 autograd
  through the whole model, and a 0/1 tensor feed against the NumPy feed.
"""
import collections

import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests import dense_adjacency_oracle as DA
from tests import test_canaries_cpu as K

pytestmark = pytest.mark.gpu

FWD_BARS = {"fp32": 1e-5, "bf16x3": 1e-4, "bf16": 2e-2}
DROP_SEED = 2718
TAG = " [dense adjacency on the device]"
REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}

Case = collections.namedtuple("Case", "D precision T b v steps bias keep cell layers residual")


def case(D, precision, T=4, b=6, v=29, steps=3, bias=True, keep=1.0, cell="GRU", layers=None, residual=False):
    return Case(D, precision, T, b, v, steps, bias, keep, cell, layers, residual)


def params(c):
    layers = c.layers or [c.steps]
    return {"hidden_size": c.D, "layer_timesteps": layers, "residual_connections": {"1": [0]} if c.residual and len(layers) > 1 else {},
            "use_edge_bias": c.bias, "use_edge_msg_avg_aggregation": False, "graph_rnn_cell": c.cell,
            "graph_rnn_activation": "relu" if c.cell == "RNN" else "tanh"}


def layer_weights(c, seed=3):
    p = params(c)
    if c.cell == "GRU" and len(p["layer_timesteps"]) == 1:   # the dense model's weights (dense:84-91), bias [T, D]
        w = O.init_dense_weights(p, c.T, np.random.default_rng(seed))
        return [{k: (v.reshape(c.T, c.D) if k == "edge_biases" else v) for k, v in w.items()}]
    w = O.init_sparse_weights(p, c.T, np.random.default_rng(seed), edge_bias_scale=0.1)
    return [{k: (v.reshape(c.T, c.D) if k == "edge_biases" else v) for k, v in lw.items()} for lw in w]


def matrix(kind, b, T, v, seed=0):
    rng = np.random.default_rng(seed + 17)
    if kind == "binary":
        A = (rng.random((b, T, v, v)) < min(1.0, 2.5 / max(v, 1))).astype(np.float32)
    elif kind == "soft":   # a row softmax of random scores: every entry nonzero
        s = rng.normal(0, 1, (b, T, v, v))
        e = np.exp(s - s.max(-1, keepdims=True))
        A = (e / e.sum(-1, keepdims=True)).astype(np.float32)
    elif kind == "negative":
        A = rng.normal(0, 0.4, (b, T, v, v)).astype(np.float32)
        A[rng.random(A.shape) < 0.5] = 0.0
    elif kind == "zero":
        A = np.zeros((b, T, v, v), np.float32)
    elif kind == "scaled":   # per-graph scales from 1e-3 to 1e3
        s = rng.normal(0, 1, (b, T, v, v))
        e = np.exp(s - s.max(-1, keepdims=True))
        A = e / e.sum(-1, keepdims=True) * np.logspace(-3, 3, b)[:, None, None, None]
        A = A.astype(np.float32)
    else:
        raise ValueError(kind)
    return A


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


class Run:
    """An engine holding a dense-device batch of case ``c`` with its matrix set."""

    def __init__(self, c, kind="soft", save=False, det=False, bwd="fp32", A=None, seed=0):
        from gated_graph_neural_network_samples_b200.engine import PropagationEngine
        self.c = c
        self.A = matrix(kind, c.b, c.T, c.v, seed) if A is None else A
        self.h0 = np.random.default_rng(seed + 5).normal(0, 0.5, (c.b * c.v, c.D)).astype(np.float32)
        self.w = layer_weights(c)
        self.eng = PropagationEngine(params(c), c.T, precision=c.precision)
        self.eng.set_deterministic(det)
        self.eng.set_backward_precision(bwd)
        if c.keep < 1.0:
            self.eng.set_state_dropout(c.keep, DROP_SEED)
        self.dev_w = [{REN.get(k, k): _cuda(v) for k, v in lw.items()} for lw in self.w]
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(save)
        self.g = self.eng.prepare_graph_dense_device(c.b, c.v)
        self.eng.set_graph_prepared(self.g)
        assert self.eng.plan.endswith(TAG), self.eng.plan
        assert ("STREAM" in self.eng.plan) == (c.precision != "fp32") and ("stepwise" in self.eng.plan) == (c.precision == "fp32")
        assert self.eng.num_messages() == c.b * c.T * c.v * c.v
        self.tA = _cuda(self.A)
        self.eng.set_message_weights(self.tA)
        self.th0 = _cuda(self.h0)

    def forward(self):
        self.out = self.eng.forward(self.th0)
        self.eng.sync_check()
        return self.out.cpu().numpy()

    def reference(self, A=None, requires_grad=False, g_out=None):
        """float64 (out, and with g_out: d h0, per-layer grads keyed as the engine's, dA)."""
        import torch
        drop = (self.c.keep, DROP_SEED) if self.c.keep < 1.0 else None
        h0 = torch.tensor(self.h0, dtype=torch.float64, requires_grad=g_out is not None)
        At = torch.tensor(self.A if A is None else A, dtype=torch.float64, requires_grad=g_out is not None)
        ws = [{k: torch.tensor(v, dtype=torch.float64, requires_grad=g_out is not None) for k, v in lw.items()} for lw in self.w]
        out = DA.propagation_torch(h0, At, ws, params(self.c), state_dropout=drop)
        if g_out is None:
            return out.detach().numpy()
        (out * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
        return (out.detach().numpy(), h0.grad.numpy(), [{REN.get(k, k): t.grad.numpy() for k, t in lw.items()} for lw in ws], At.grad.numpy())

    def backward(self, g_out, with_dA=True):
        import torch
        grads = [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in self.dev_w]
        dh0 = torch.zeros_like(self.th0)
        dA = torch.zeros_like(self.tA) if with_dA else None
        self.eng.backward(_cuda(g_out), grads, dh0, d_message_weights=dA)
        self.eng.sync_check()
        return (dh0.cpu().numpy(), [{k: t.cpu().numpy() for k, t in lw.items()} for lw in grads], None if dA is None else dA.cpu().numpy())


def _check_forward(c, kind, per_graph=False):
    r = Run(c, kind)
    got = r.forward()
    ref = r.reference()
    assert np.all(np.isfinite(got)), (c, kind)
    if per_graph:
        for g in range(c.b):
            rows = slice(g * c.v, (g + 1) * c.v)
            err = U.max_rel_err(got[rows], ref[rows])
            assert err < FWD_BARS[c.precision], (c, kind, g, err)
    else:
        err = U.max_rel_err(got, ref)
        print("\nDENSE-DEV %s %-8s %.3e  %s" % (c, kind, err, r.eng.plan))
        assert err < FWD_BARS[c.precision], (c, kind, err)
    return r


# ---------------------------------------------------------------------------------------------------------------- forward
FORWARD = [case(D, p) for D in (4, 100, 128, 132, 256, 512) for p in ("fp32", "bf16x3")] + [case(100, "bf16"), case(512, "bf16")]


@pytest.mark.parametrize("c", FORWARD, ids=lambda c: "%s-%d" % (c.precision, c.D))
def test_forward_against_the_dense_loops(c):
    """The reference's own dense loops (oracle.dense_propagation_loops) on a soft matrix, one GRU layer."""
    r = Run(c, "soft")
    got = r.forward()
    w = dict(r.w[0])
    if "edge_biases" in w:
        w["edge_biases"] = w["edge_biases"].reshape(c.T, 1, c.D)
    ref = O.dense_propagation_loops(r.h0.reshape(c.b, c.v, c.D), r.A, w, {"num_timesteps": c.steps, "use_edge_bias": c.bias}).reshape(-1, c.D)
    err = U.max_rel_err(got, ref)
    print("\nDENSE-DEV loops %s-%d %.3e  %s" % (c.precision, c.D, err, r.eng.plan))
    assert err < FWD_BARS[c.precision], err


@pytest.mark.parametrize("kind", ["binary", "soft", "negative", "zero"])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("D", [100, 256])
def test_forward_matrix_kinds(kind, precision, D):
    _check_forward(case(D, precision), kind)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_forward_per_graph_scales(precision):
    """Graphs scaled from 1e-3 to 1e3, each held to the bar against its own largest state.  A ReLU RNN keeps every graph's states in
    proportion to its scale; a GRU would saturate the large graphs and pass the small ones' absolute error through at full size."""
    _check_forward(case(128, precision, b=7, cell="RNN", layers=[2]), "scaled", per_graph=True)


@pytest.mark.parametrize("T,v", [(1, 1), (1, 29), (32, 29), (4, 128), (4, 300), (32, 1)])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_forward_shapes(T, v, precision):
    b = 3 if v >= 128 else 6
    _check_forward(case(132, precision, T=T, b=b, v=v, steps=2), "soft")


@pytest.mark.parametrize("c", [case(100, "bf16x3", keep=0.8), case(256, "fp32", keep=0.8, bias=False), case(100, "fp32", bias=False),
                               case(256, "bf16x3", cell="RNN", layers=[2, 1], residual=True)],
                         ids=["dropout-bf16x3", "dropout-nobias-fp32", "nobias-fp32", "rnn-residual-bf16x3"])
def test_forward_options(c):
    _check_forward(c, "negative")


def test_empty_batch():
    import torch
    for precision in ("fp32", "bf16x3"):
        c = case(100, precision, b=0)
        r = Run(c, A=np.zeros((0, 4, 29, 29), np.float32), save=True)
        out = r.eng.forward(torch.zeros(0, 100, device="cuda"))
        r.eng.sync_check()
        assert out.shape == (0, 100)


# ---------------------------------------------------------------------------------------------------------------- gradients
GRADS = [case(100, "fp32"), case(260, "fp32", b=4), case(100, "bf16x3"), case(512, "bf16x3", b=3), case(132, "bf16x3", keep=0.8),
         case(256, "fp32", cell="RNN", layers=[2, 1], residual=True, b=4), case(128, "bf16x3", bias=False, T=1)]


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("c", GRADS, ids=lambda c: "%s-%d-%s-keep%s" % (c.precision, c.D, c.cell, c.keep))
def test_gradients_against_float64_autograd(c, bwd):
    r = Run(c, "negative", save=True, bwd=bwd)
    r.forward()
    g = np.random.default_rng(7).normal(0, 1, r.h0.shape).astype(np.float32)
    dh0, gw, dA = r.backward(g)
    _, rdh0, rgw, rdA = r.reference(g_out=g)
    bar = 2.5e-5 if c.precision == "fp32" and bwd == "fp32" else 2e-4
    errs = {"dh0": U.max_rel_err(dh0, rdh0), "dA": U.max_rel_err(dA, rdA)}
    for l, (a, ref) in enumerate(zip(gw, rgw)):
        for k in ref:
            errs["%d/%s" % (l, k)] = U.max_rel_err(a[k].reshape(ref[k].shape), ref[k])
    print("\nDENSE-DEV grads %s bwd=%s %s" % (c, bwd, " ".join("%s=%.2e" % kv for kv in errs.items())))
    assert all(e < bar for e in errs.values()), errs


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("c", [case(100, "fp32"), case(256, "bf16x3")], ids=["fp32-100", "bf16x3-256"])
def test_gradients_repeat_bit_for_bit(c, det):
    """dA and d h0 repeat their bits in both deterministic modes (no atomics in their kernels); the weight gradients do in deterministic
    mode, whose fixed-order sums they take (outside it they are added with float atomics, as on every batch kind)."""
    g = np.random.default_rng(8).normal(0, 1, (c.b * c.v, c.D)).astype(np.float32)
    results = []
    for fresh in (False, True):
        r = Run(c, "soft", save=True, det=det)
        r.forward()
        results.append(r.backward(g))
        if not fresh:
            results.append(r.backward(g))
    for other in results[1:]:
        np.testing.assert_array_equal(other[0], results[0][0])
        np.testing.assert_array_equal(other[2], results[0][2])
        if not det:
            continue
        for a, b in zip(other[1], results[0][1]):
            for k in a:
                np.testing.assert_array_equal(a[k], b[k], err_msg=k)


@pytest.mark.parametrize("D", [260, 512])
def test_fp32_binary_matrix_is_bit_identical_to_set_graph_dense(D):
    """Both paths run the per-timestep fp32 plan with one summation order: fmaf(0, x, acc) leaves acc as it is, fmaf(1, x, acc) = acc + x."""
    import torch
    c = case(D, "fp32", b=5)
    r = Run(c, "binary", save=True, det=True)
    got = r.forward()
    g = np.random.default_rng(9).normal(0, 1, r.h0.shape).astype(np.float32)
    dh0, gw, _ = r.backward(g)
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(params(c), c.T, precision="fp32")
    eng.set_deterministic(True)
    eng.set_weights(r.dev_w)
    eng.set_save_for_backward(True)
    eng.set_graph_dense(r.A)
    assert "stepwise" in eng.plan, eng.plan
    out = eng.forward(r.th0)
    grads = [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in r.dev_w]
    dh0_ref = torch.zeros_like(r.th0)
    eng.backward(_cuda(g), grads, dh0_ref)
    eng.sync_check()
    np.testing.assert_array_equal(got, out.cpu().numpy())
    np.testing.assert_array_equal(dh0, dh0_ref.cpu().numpy())
    for a, b in zip(gw, grads):
        for k in a:
            np.testing.assert_array_equal(a[k], b[k].cpu().numpy(), err_msg=k)


# ---------------------------------------------------------------------------------------------------------------- lifecycle
def test_lifecycle():
    import torch
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    c = case(132, "bf16x3")
    r = Run(c, "soft", save=True)
    r.eng.set_graph_prepared(r.g)                       # an upload forgets the matrix
    with pytest.raises(GgnnError, match="set_message_weights"):
        r.eng.forward(r.th0)
    r.eng.set_message_weights(r.tA)
    first = r.forward()
    assert U.max_rel_err(first, r.reference()) < FWD_BARS[c.precision]
    r.eng.set_message_weights(r.tA)                     # a re-set drops the saved activations
    g = np.zeros(r.h0.shape, np.float32)
    with pytest.raises(GgnnError):
        r.eng.backward(_cuda(g), [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in r.dev_w], torch.zeros_like(r.th0),
                       d_message_weights=torch.zeros_like(r.tA))
    A2 = matrix("negative", c.b, c.T, c.v, seed=3)     # a new matrix on the same prepared batch: no re-prepare
    r.eng.set_message_weights(_cuda(A2))
    second = r.forward()
    assert U.max_rel_err(second, r.reference(A=A2)) < FWD_BARS[c.precision]
    assert U.max_rel_err(second, first) > 1e-3


# ---------------------------------------------------------------------------------------------------------------- canaries
@pytest.mark.parametrize("c", [case(100, "fp32", b=5, v=40), case(132, "bf16x3", b=5, v=40)], ids=["fp32", "bf16x3"])
def test_nan_graphs_do_not_reach_clean_ones(c):
    """Graphs 1 and 3 get payload NaN in every h0 row and every matrix entry: the other graphs keep their bits and stay finite."""
    clean = Run(c, "soft", seed=1)
    out_clean = clean.forward()
    A = clean.A.copy()
    h0 = clean.h0.copy()
    bad = np.zeros(c.b * c.v, bool)
    for g in (1, 3):
        A[g] = K.payload_nan(A[g].shape)
        bad[g * c.v:(g + 1) * c.v] = True
    h0[bad] = K.payload_nan(h0[bad].shape)
    r = Run(c, A=A, seed=1)
    r.th0 = _cuda(h0)
    out = r.forward()
    assert np.all(np.isfinite(out[~bad]))
    np.testing.assert_array_equal(out[~bad], out_clean[~bad])


@pytest.mark.parametrize("c", [case(100, "fp32", b=5, v=37), case(260, "fp32", b=3, v=37), case(132, "bf16x3", b=5, v=37)],
                         ids=["fp32-100", "fp32-260", "bf16x3-132"])
def test_guard_bands_around_the_matrix_and_every_buffer(c):
    """The matrix, h0, h_out, d_out, d h0, every weight gradient and dA between payload-NaN bands: the plain buffers' bits, no payload
    word in an output, both bands intact."""
    import torch
    base = Run(c, "negative", save=True, det=True)
    g = np.random.default_rng(3).normal(0, 1, base.h0.shape).astype(np.float32)
    rng = np.random.default_rng(4)
    preA = rng.normal(0, 1, base.A.shape).astype(np.float32)

    def run(guard):
        keep = []

        def buf(shape, fill=None):
            if not guard:
                return (_cuda(fill) if fill is not None else torch.empty(shape, device="cuda")).reshape(shape)
            n = int(np.prod(shape))
            gb = K.guarded(n)
            if fill is not None:
                gb.view.copy_(_cuda(np.asarray(fill, np.float32).reshape(-1)))
            keep.append(gb)
            return gb.view.view(*shape)
        r = base.eng.__class__(params(c), c.T, precision=c.precision)
        r.set_deterministic(True)
        r.set_weights(base.dev_w)
        r.set_save_for_backward(True)
        r.set_graph_prepared(r.prepare_graph_dense_device(c.b, c.v))
        r.set_message_weights(buf(base.A.shape, base.A))
        out = buf(base.h0.shape)
        r.forward(buf(base.h0.shape, base.h0), out)
        grads = [{k: buf(tuple(t.shape), np.zeros(tuple(t.shape), np.float32)) for k, t in lw.items()} for lw in base.dev_w]
        dh0 = buf(base.h0.shape)
        dA = buf(base.A.shape, preA)
        r.backward(buf(base.h0.shape, g), grads, dh0, d_message_weights=dA)
        r.sync_check()
        outs = [out, dh0, dA] + [t for lw in grads for t in lw.values()]
        if guard:
            assert not any(K.has_payload(t) for t in outs)
            assert all(b.bands_intact() for b in keep)
        return [t.cpu().numpy() for t in outs]
    for a, b in zip(run(True), run(False)):
        np.testing.assert_array_equal(a, b)


# ---------------------------------------------------------------------------------------------------------------- the plug-in
def _model(tmp_path, precision, seed=0):
    import torch
    from gated_graph_neural_network_samples_b200 import chem_dense, synthetic
    torch.manual_seed(seed)
    np.random.seed(seed)
    mols = synthetic.make_molecules(24, seed=6)
    return chem_dense.DenseGGNNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:16],
                                          "--valid_data": mols[16:], "--config": {"hidden_size": 32, "batch_size": 8, "num_timesteps": 2,
                                                                                  "random_seed": seed}})


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_plugin_learned_scale_gradient_and_binary_feed(tmp_path, precision):
    """Two training steps of DenseGGNNChemModel on A' = A * s[t] with a learnable per-type scale s: each step's d s matches float64
    autograd through the whole model (propagation, readout, loss), then Adam steps the model.  A 0/1 tensor feed gives the NumPy feed's
    loss within the forward bar."""
    import torch
    m = _model(tmp_path, precision)
    m.make_train_step()
    s = torch.tensor([0.7, 1.3, 0.9, 1.1], device="cuda", requires_grad=True)
    T, D = 4, 32
    for feed in list(m.make_minibatch_iterator(m.train_data, True))[:2]:
        feed = dict(feed)
        feed.pop("_prepared_graph", None)
        feed["graph_state_keep_prob"] = feed["edge_weight_dropout_keep_prob"] = 1.0
        adj = np.asarray(feed["adjacency_matrix"], np.float32)
        with torch.no_grad():
            loss_np = float(m.forward_batch(dict(feed))[0])
            loss_01 = float(m.forward_batch(dict(feed, adjacency_matrix=torch.from_numpy(adj).cuda()))[0])
        assert abs(loss_01 - loss_np) <= FWD_BARS[precision] * abs(loss_np), (loss_01, loss_np)
        loss = m.forward_batch(dict(feed, adjacency_matrix=torch.from_numpy(adj).cuda() * s.view(1, -1, 1, 1)))[0]
        got = torch.autograd.grad(loss, s, retain_graph=True)[0].cpu().numpy()
        # float64 autograd of the same model
        s64 = s.detach().cpu().double().requires_grad_(True)
        f64 = lambda t: t.detach().cpu().double()
        wts = {"edge_weights": f64(m.weights["edge_weights"]), "edge_biases": f64(m.weights["edge_biases"]).reshape(T, D)}
        wts.update({k: f64(v) for k, v in m.weights["node_gru"].items()})
        h0 = f64(m.initial_node_representation_tensor()).reshape(-1, D)
        p = {"hidden_size": D, "layer_timesteps": [2], "residual_connections": {}, "use_edge_bias": True, "graph_rnn_cell": "GRU",
             "graph_rnn_activation": "tanh"}
        b, v = adj.shape[0], adj.shape[2]
        final = DA.propagation_torch(h0, torch.from_numpy(adj).double() * s64.view(1, -1, 1, 1), [wts], p).reshape(b, v, D)
        tv, tm = (torch.as_tensor(np.asarray(feed[k], np.float64)) for k in ("target_values", "target_mask"))
        ref_loss = 0
        for internal_id, task_id in enumerate(m.params["task_ids"]):
            gate, trans = m.weights["regression_gate_task%i" % task_id], m.weights["regression_transform_task%i" % task_id]
            computed = O.gated_regression_torch(final, h0.reshape(b, v, D), f64(gate.weights[0]), f64(gate.biases[0]), f64(trans.weights[0]),
                                                f64(trans.biases[0]), node_mask=np.asarray(feed["node_mask"], np.float64), dtype=torch.float64)
            diff = (computed - tv[internal_id]) * tm[internal_id]
            ref_loss = ref_loss + (0.5 * diff * diff).sum() / (tm[internal_id].sum() + O.SMALL_NUMBER)
        ref_loss.backward()
        assert abs(float(loss) - float(ref_loss)) <= FWD_BARS[precision] * 10 * abs(float(ref_loss)), (float(loss), float(ref_loss))
        err = U.max_rel_err(got, s64.grad.numpy())
        print("\nDENSE-DEV plug-in %s d s %s vs %s err %.2e" % (precision, got, s64.grad.numpy(), err))
        assert err < 2e-4, err
        m.train_step(loss)                       # the model's own step: backward through the engine, clipping, Adam
        with torch.no_grad():
            s -= 0.05 * s.grad
        s.grad = None
