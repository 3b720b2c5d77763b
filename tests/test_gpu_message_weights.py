"""GPU: message weights in the sparse GGNN model against float64 (tests/message_weights_oracle.py).

A batch prepared with ``prepare_graph_sparse_weighted`` takes its weights on the device (``set_message_weights``) and scales message m's
state term by w_m on every forward plan; ``backward(..., d_message_weights=)`` adds their gradient.  Bars, max|err| / max|ref|: 1e-4 on
the forward and 2e-4 on every gradient at fp32 / bf16x3, 2e-2 at bf16.  Covered here:

* forward on every plan: fp32 FFMA variants 0 and 1 (LOCAL, GLOBAL), the per-timestep fp32 path at 260 and 512, the tile-local wgmma kernel
  (compact and 128-row tiles, GLOBAL for a 200-node component), streaming at 132, 256 and 512 (and bf16), CudnnCompatibleGRUCell on the
  tensor cores; GRU, RNN, residual inputs, edge bias, mean aggregation and state dropout;
* value independence: two weight vectors on one uploaded batch, a lone message going from 1.0 to 0.5 on the streaming plan;
* refusals: a forward before the weights, weights on an unweighted batch, an upload forgetting them, d w on an unweighted batch, a GCN
  engine, attention;
* gradients of d w, d h0 and every weight at both backward precisions, d w bit-identical across two calls in both deterministic modes;
* edge cases: zero, negative and duplicate weights, self-loops, isolated nodes, empty types, 1 and 17 edge types, the 100 000-node batch;
* memory canaries: guard bands around the weights and their gradient, and a NaN component that leaves the other components' results alone;
* an end-to-end torch run: a learned gate w = sigmoid(f . theta) through ``chem_sparse.propagate`` and a readout, theta's gradient against
  float64 autograd.
"""
import collections

import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests import message_weights_oracle as MW

pytestmark = pytest.mark.gpu

FWD_BARS = {"fp32": 1e-4, "bf16x3": 1e-4, "bf16": 2e-2}
GRAD_BAR = 2e-4
DROP_SEED = 31337
TAG = " [message-weighted]"

Case = collections.namedtuple("Case", "name D precision cell act layers residual bias avg keep env pattern batch cudnn_tc T")


def case(name, D, precision, pattern, cell="GRU", act="tanh", layers=(2, 1), residual=True, bias=True, avg=True, keep=1.0, env=None,
         batch="mol", cudnn_tc=False, T=4):
    return Case(name, D, precision, cell, act, list(layers), residual, bias, avg, keep, env or {}, pattern, batch, cudnn_tc, T)


CASES = {c.name: c for c in [
    case("ffma-v0-local", 100, "fp32", r"^fp32-ffma LOCAL\(.*colsplit=1", env={"GGNN_FFMA_VARIANT": "0"}),
    case("ffma-v1-local", 100, "fp32", r"^fp32-ffma LOCAL\(.*colsplit=2", env={"GGNN_FFMA_VARIANT": "1"}, batch="small"),
    case("ffma-v0-global", 64, "fp32", r"^fp32-ffma GLOBAL\(.*colsplit=1", env={"GGNN_FFMA_VARIANT": "0", "GGNN_FORCE_GLOBAL": "1"}),
    case("ffma-v1-global", 36, "fp32", r"^fp32-ffma GLOBAL\(.*colsplit=2", env={"GGNN_FFMA_VARIANT": "1", "GGNN_FORCE_GLOBAL": "1"}),
    case("step-260", 260, "fp32", r"^fp32-stepwise "),
    case("step-512", 512, "fp32", r"^fp32-stepwise ", layers=(2,), residual=False),
    case("tc-compact", 100, "bf16x3", r"^wgmma-bf16x3 LOCAL\(.*compact", batch="small"),
    case("tc-128row", 128, "bf16x3", r"^wgmma-bf16x3 LOCAL\(.*rows/tile<=128 DP", batch="many", layers=(2,), residual=False),
    case("tc-global-200", 100, "bf16x3", r"^wgmma-bf16x3 GLOBAL\(", batch="big"),
    case("stream-132", 132, "bf16x3", r"^wgmma-bf16x3 STREAM\("),
    case("stream-256", 256, "bf16x3", r"^wgmma-bf16x3 STREAM\("),
    case("stream-512", 512, "bf16x3", r"^wgmma-bf16x3 STREAM\(", layers=(2,), residual=False),
    case("stream-256-bf16", 256, "bf16", r"^wgmma-bf16 STREAM\("),
    case("cudnn-tc", 100, "bf16x3", r"^wgmma-bf16x3 STREAM\+cudnn-gru", cell="CudnnCompatibleGRUCell", cudnn_tc=True),
    case("rnn-relu-fp32", 100, "fp32", r"^fp32-ffma ", cell="RNN", act="relu", bias=False),
    case("rnn-relu-stream", 256, "bf16x3", r"^wgmma-bf16x3 STREAM\(", cell="RNN", act="relu", avg=False),
    case("dropout-tc", 100, "bf16x3", r"^wgmma-bf16x3 LOCAL\(", keep=0.8),
    case("dropout-stream", 256, "bf16x3", r"^wgmma-bf16x3 STREAM\(", keep=0.8, bias=False),
    case("plain-fp32", 100, "fp32", r"^fp32-ffma ", bias=False, avg=False, residual=False, layers=(3,)),
]}
EDGE = {c.name: c for c in [
    case("edges-fp32", 100, "fp32", r"^fp32-ffma ", batch="edges"),
    case("edges-tc", 100, "bf16x3", r"^wgmma-bf16x3 LOCAL\(", batch="edges"),
    case("edges-stream", 256, "bf16x3", r"^wgmma-bf16x3 STREAM\(", batch="edges"),
    case("t1-tc", 100, "bf16x3", r"^wgmma-bf16x3 LOCAL\(", T=1),
    case("t17-fp32", 64, "fp32", r"^fp32-ffma ", T=17),
    case("t17-stream", 256, "bf16x3", r"^wgmma-bf16x3 STREAM\(", T=17, layers=(1,), residual=False),
]}
GRAD_CASES = ("ffma-v0-local", "step-260", "tc-compact", "tc-global-200", "stream-256", "cudnn-tc", "rnn-relu-stream", "dropout-tc")


def params(c):
    p = {"hidden_size": c.D, "layer_timesteps": c.layers, "residual_connections": {"1": [0]} if c.residual and len(c.layers) > 1 else {},
         "use_edge_bias": c.bias, "use_edge_msg_avg_aggregation": c.avg, "graph_rnn_cell": c.cell, "graph_rnn_activation": c.act}
    return p


def _indeg(adj, V, T):
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return indeg


def make_batch(kind, D, T, seed=0):
    """(adjacency lists, in-degrees, h0) of a batch kind: molecules, a few (small) or many molecules, a 200-node component beside
    molecules, or the edge-case batch (self-loops, duplicate messages, isolated nodes, an empty type, a hub of 12 messages)."""
    rng = np.random.default_rng(seed + 11)
    if kind in ("mol", "small", "many", "edges"):
        n = {"mol": 40, "small": 12, "many": 1500, "edges": 20}[kind]
        _, b = U.molecule_batch(n, D, T, seed)
        adj = [np.asarray(a, np.int32).reshape(-1, 2) for a in b["adjacency_lists"]]
        V = b["initial_node_representation"].shape[0]
        if kind == "edges":
            adj[0] = np.concatenate([adj[0], [[5, 5], [6, 6], [1, 2], [1, 2], [1, 2]], [[s, 0] for s in range(1, 13)]]).astype(np.int32)
            if T > 1:
                adj[T - 1] = np.zeros((0, 2), np.int32)   # an empty type
            V += 7                                        # isolated nodes at the end
        h0 = rng.normal(0, 0.5, (V, D)).astype(np.float32)
    else:   # "big": a 200-node connected component (a path plus 200 random chords) and 10 molecules behind it
        n = 200
        pairs = [(i, i + 1) for i in range(n - 1)] + [tuple(sorted(rng.choice(n, 2, replace=False))) for _ in range(n)]
        _, b = U.molecule_batch(10, D, T, seed)
        mol = [np.asarray(a, np.int32).reshape(-1, 2) + n for a in b["adjacency_lists"]]
        adj = []
        for t in range(T):
            mine = np.array([p for k, p in enumerate(pairs) if k % T == t], np.int32).reshape(-1, 2)
            adj.append(np.concatenate([mine, mine[:, ::-1], mol[t]]).astype(np.int32))
        V = n + b["initial_node_representation"].shape[0]
        h0 = rng.normal(0, 0.5, (V, D)).astype(np.float32)
    return adj, _indeg(adj, V, T), h0


def draw_weights(M, regime="uniform", seed=0):
    rng = np.random.default_rng(seed + 5)
    if regime == "uniform":
        return rng.uniform(0.25, 1.75, M).astype(np.float32)
    w = rng.normal(0, 1.0, M).astype(np.float32)   # "signed": zeros, negatives and ones among them
    w[::7] = 0.0
    w[3::11] = 1.0
    return w


def layer_weights(c, seed=3):
    p = params(c)
    w = O.init_sparse_weights(p, c.T, np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 1)
    for lw in w:   # nonzero candidate biases
        for k in ("cand_bias", "rnn_bias"):
            if k in lw:
                lw[k] = rng.normal(0, 0.1, lw[k].shape).astype(np.float32)
    return w


def engine_for(c, det=False, bwd="fp32"):
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(params(c), c.T, precision=c.precision, cudnn_gru_tensor_cores=c.cudnn_tc)
    eng.set_deterministic(det)
    eng.set_backward_precision(bwd)
    if c.keep < 1.0:
        eng.set_state_dropout(c.keep, DROP_SEED)
    return eng


def _env(monkeypatch, env):
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM", "GGNN_FFMA_VARIANT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


class Run:
    """An engine holding a message-weighted batch of case ``c`` with its weights set."""

    def __init__(self, c, monkeypatch, regime="uniform", save=False, det=False, bwd="fp32", batch=None, mw=None):
        import re
        _env(monkeypatch, c.env)
        self.c = c
        self.adj, self.indeg, self.h0 = batch or make_batch(c.batch, c.D, c.T)
        self.M = sum(a.shape[0] for a in self.adj)
        self.mw = draw_weights(self.M, regime) if mw is None else mw
        self.w = layer_weights(c)
        self.eng = engine_for(c, det, bwd)
        self.dev_w = U.to_cuda_weights(self.w)
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(save)
        self.g = self.eng.prepare_graph_sparse_weighted(self.adj, self.indeg)
        self.eng.set_graph_prepared(self.g)
        assert self.eng.plan.endswith(TAG) and re.search(c.pattern, self.eng.plan), (c.name, self.eng.plan)
        assert self.eng.num_messages() == self.M
        self.eng.set_message_weights(_cuda(self.mw))
        self.th0 = _cuda(self.h0)

    def forward(self):
        out = self.eng.forward(self.th0)
        self.eng.sync_check()
        self.out = out
        return out.cpu().numpy()

    def reference(self, mw=None):
        import torch
        drop = (self.c.keep, DROP_SEED) if self.c.keep < 1.0 else None
        return MW.propagation_torch(self.h0, self.adj, self.indeg, self.w, params(self.c), self.mw if mw is None else mw, dtype=torch.float64,
                                    state_dropout=drop).numpy()

    def backward(self, g_out):
        import torch
        grads = [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in self.dev_w]
        dh0 = torch.zeros_like(self.th0)
        dmw = torch.zeros(self.M, dtype=torch.float32, device="cuda")
        self.eng.backward(_cuda(g_out), grads, dh0, d_message_weights=dmw)
        self.eng.sync_check()
        return dmw.cpu().numpy(), dh0.cpu().numpy(), [{k: t.cpu().numpy() for k, t in lw.items()} for lw in grads]


def _forward_case(c, monkeypatch, regime="uniform"):
    r = Run(c, monkeypatch, regime)
    got = r.forward()
    err = U.max_rel_err(got, r.reference())
    print("\nMSGW %-20s %-8s %.3e  %s" % (c.name, regime, err, r.eng.plan))
    assert np.all(np.isfinite(got)) and err < FWD_BARS[c.precision], (c.name, regime, err)
    return r


# ---------------------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("name", sorted(CASES))
def test_forward_matches_float64(name, monkeypatch):
    _forward_case(CASES[name], monkeypatch)


@pytest.mark.parametrize("name", sorted(EDGE))
@pytest.mark.parametrize("regime", ["uniform", "signed"])
def test_edge_cases(name, regime, monkeypatch):
    _forward_case(EDGE[name], monkeypatch, regime)


@pytest.mark.parametrize("name", ["ffma-v0-local", "tc-compact", "stream-256"])
def test_all_ones_is_the_unweighted_model(name, monkeypatch):
    """Weights of exactly 1.0 give the unweighted batch's forward (to float tolerance: the streaming plan sums every pair as a virtual row)."""
    c = CASES[name]
    r = Run(c, monkeypatch)
    r.eng.set_message_weights(_cuda(np.ones(r.M, np.float32)))
    got = r.forward()
    plain = r.eng.__class__(params(c), c.T, precision=c.precision)
    plain.set_weights(r.dev_w)
    plain.set_graph_sparse(r.adj, r.indeg)
    ref = plain.forward(r.th0).cpu().numpy()
    assert U.max_rel_err(got, ref) < 1e-5, U.max_rel_err(got, ref)
    assert U.max_rel_err(got, O.sparse_propagation_loops(r.h0, r.adj, r.indeg, r.w, params(c))) < FWD_BARS[c.precision]


@pytest.mark.parametrize("name", ["tc-compact", "stream-256", "ffma-v1-local"])
def test_two_weight_vectors_on_one_upload(name, monkeypatch):
    """One upload, two weight vectors: each forward matches its own oracle.  A (target, type) pair with one message weighs 1.0 first and
    0.5 then -- the streaming plan made it a virtual row at prepare time, whatever its weight."""
    c = CASES[name]
    adj, indeg, h0 = make_batch(c.batch, c.D, c.T)
    M = sum(a.shape[0] for a in adj)
    _, tgt, typ = O.message_arrays(adj)
    key = tgt.astype(np.int64) * c.T + typ
    lone = int(np.nonzero(np.bincount(key, minlength=int(key.max()) + 1)[key] == 1)[0][0])
    w1 = draw_weights(M, "uniform", seed=1)
    w1[lone] = 1.0
    w2 = draw_weights(M, "signed", seed=2)
    w2[lone] = 0.5
    r = Run(c, monkeypatch, batch=(adj, indeg, h0), mw=w1)
    for w in (w1, w2):
        r.eng.set_message_weights(_cuda(w))
        got = r.forward()
        err = U.max_rel_err(got, r.reference(w))
        assert err < FWD_BARS[c.precision], (name, err)
    if r.g.info()["streaming"]:
        rows = np.count_nonzero(np.diff(r.g.arrays(c.T)["row_ptr"]))
        assert r.g.stream_tables()["vrow_ptr"].shape[0] - 1 == rows


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_refusals(monkeypatch):
    import ctypes as C
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine, GgnnError, PropagationEngine
    c = CASES["tc-compact"]
    adj, indeg, h0 = make_batch("small", c.D, c.T)
    M = sum(a.shape[0] for a in adj)
    eng = engine_for(c)
    eng.set_weights(U.to_cuda_weights(layer_weights(c)))
    eng.set_save_for_backward(True)
    g = eng.prepare_graph_sparse_weighted(adj, indeg)
    eng.set_graph_prepared(g)
    th0 = _cuda(h0)
    with pytest.raises(GgnnError) as e:
        eng.forward(th0)
    assert e.value.code == -3
    eng.set_message_weights(_cuda(np.ones(M)))
    eng.forward(th0)
    eng.set_graph_prepared(g)   # an upload forgets the weights
    with pytest.raises(GgnnError) as e:
        eng.forward(th0)
    assert e.value.code == -3
    eng.set_graph_sparse(adj, indeg)   # an unweighted batch takes no weights, and no d w
    with pytest.raises(GgnnError) as e:
        eng.set_message_weights(_cuda(np.ones(M)))
    assert e.value.code == -3
    out = eng.forward(th0)
    grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in U.to_cuda_weights(layer_weights(c))]
    with pytest.raises(GgnnError) as e:
        eng.backward(torch.ones_like(out), grads, None, d_message_weights=torch.zeros(M, device="cuda"))
    assert e.value.code == -3
    with pytest.raises(GgnnError):
        eng.set_message_weights(_cuda(np.ones(M + 1)))
    # a GCN engine: GGNN_ESTATE; attention: GGNN_EUNSUPPORTED
    gcn = GCNEngine(100, 2, precision="bf16x3")
    T = len(adj)
    ptrs = (C.c_void_p * T)(*[a.ctypes.data for a in adj])
    counts = (C.c_int32 * T)(*[a.shape[0] for a in adj])
    h = C.c_void_p()
    rc = gcn.lib.ggnn_prepare_graph_sparse_weighted(gcn._h, 0, indeg.shape[0], ptrs, counts, indeg.ctypes.data, C.byref(h))
    assert rc == -3
    gcn.lib.ggnn_free_prepared_graph(h)
    att = PropagationEngine(dict(params(c), use_propagation_attention=True), c.T, precision="bf16x3", attention_tensor_cores=True)
    with pytest.raises(GgnnError, match="attention"):
        att.prepare_graph_sparse_weighted(adj, indeg)


# ---------------------------------------------------------------------------------------------------------------- gradients
def _autograd(r, g_out):
    import torch
    tw = [{k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in lw.items()} for lw in r.w]
    th0 = torch.tensor(r.h0, dtype=torch.float64, requires_grad=True)
    tmw = torch.tensor(r.mw, dtype=torch.float64, requires_grad=True)
    drop = (r.c.keep, DROP_SEED) if r.c.keep < 1.0 else None
    out = MW.propagation_torch(th0, r.adj, r.indeg, tw, params(r.c), tmw, dtype=torch.float64, state_dropout=drop)
    (out * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
    return tmw.grad.numpy(), th0.grad.numpy(), [{k: t.grad.numpy() for k, t in lw.items()} for lw in tw]


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", GRAD_CASES)
def test_gradients_match_float64_autograd(name, bwd, monkeypatch):
    c = CASES[name]
    r = Run(c, monkeypatch, "signed", save=True, bwd=bwd)
    got = r.forward()
    g_out = np.random.default_rng(7).normal(size=got.shape).astype(np.float32)
    dmw, dh0, gw = r.backward(g_out)
    rdmw, rdh0, rgw = _autograd(r, g_out)
    REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}
    errs = [(U.max_rel_err(dmw, rdmw), "d w"), (U.max_rel_err(dh0, rdh0), "d h0")]
    for l, lw in enumerate(rgw):
        for k, ref in lw.items():
            errs.append((U.max_rel_err(gw[l][REN.get(k, k)].reshape(ref.shape), ref), "layer %d d %s" % (l, k)))
    print("\nMSGWGRAD %-16s bwd %-6s d w %.2e  worst %.2e on %s" % (name, bwd, errs[0][0], *max(errs)))
    for e, n in errs:
        assert e < GRAD_BAR, (name, bwd, n, e)


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", ["tc-compact", "stream-256", "step-260"])
def test_weight_gradient_repeats_bit_for_bit(name, bwd, det, monkeypatch):
    c = CASES[name]
    r = Run(c, monkeypatch, "signed", save=True, det=det, bwd=bwd)
    got = r.forward()
    g_out = np.random.default_rng(8).normal(size=got.shape).astype(np.float32)
    first = r.backward(g_out)
    second = r.backward(g_out)
    np.testing.assert_array_equal(first[0], second[0])
    np.testing.assert_array_equal(first[1], second[1])
    if det:
        for a, b in zip(first[2], second[2]):
            for k in a:
                np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_100k_node_batch(monkeypatch):
    """The benchmarked 100 000-node batch (hidden 100, [4] timesteps, GRU) on the tile-local wgmma kernel: forward and d w."""
    from gated_graph_neural_network_samples_b200 import workloads
    wl = workloads.build("default_batch_100k_nodes")
    c = case("100k", 100, "bf16x3", r"^wgmma-bf16x3 LOCAL\(", layers=(4,), residual=False, bias=False, avg=True)
    adj = [np.asarray(a, np.int32).reshape(-1, 2) for a in wl["adjacency_lists"]]
    r = Run(c, monkeypatch, "signed", save=True, batch=(adj, np.asarray(wl["num_incoming_edges_per_type"], np.float32),
                                                        np.asarray(wl["h0"], np.float32)))
    got = r.forward()
    assert U.max_rel_err(got, r.reference()) < FWD_BARS["bf16x3"]
    g_out = np.random.default_rng(9).normal(size=got.shape).astype(np.float32)
    dmw, dh0, _ = r.backward(g_out)
    rdmw, rdh0, _ = _autograd(r, g_out)
    assert U.max_rel_err(dmw, rdmw) < GRAD_BAR and U.max_rel_err(dh0, rdh0) < GRAD_BAR


# ---------------------------------------------------------------------------------------------------------------- canaries
def _guarded(n, fill):
    """A [n] view between two bands of 64 payload NaNs, in one allocation; the view starts as ``fill``."""
    import torch
    buf = torch.full((n + 128,), float("nan"), device="cuda")
    view = buf[64:64 + n]
    view.fill_(fill)
    return buf, view


@pytest.mark.parametrize("name", ["ffma-v0-local", "tc-compact", "stream-256", "step-260"])
def test_guard_bands(name, monkeypatch):
    """The weights and their gradient between NaN bands: the same forward bits and d w as on plain buffers, and the bands intact."""
    import torch
    c = CASES[name]
    r = Run(c, monkeypatch, "signed", save=True, det=True)
    plain = r.forward()
    g_out = np.random.default_rng(10).normal(size=plain.shape).astype(np.float32)
    dmw_plain = r.backward(g_out)[0]
    wbuf, wview = _guarded(r.M, 0.0)
    wview.copy_(_cuda(r.mw))
    r.eng.set_message_weights(wview)
    np.testing.assert_array_equal(r.forward(), plain)
    gbuf, gview = _guarded(r.M, 0.25)
    grads = [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in r.dev_w]
    r.eng.backward(_cuda(g_out), grads, None, d_message_weights=gview)
    r.eng.sync_check()
    want = (torch.from_numpy(dmw_plain) + torch.tensor(0.25)).numpy()
    np.testing.assert_array_equal(gview.cpu().numpy(), want)
    for buf in (wbuf, gbuf):
        b = buf.cpu().numpy()
        assert np.all(np.isnan(b[:64])) and np.all(np.isnan(b[-64:]))


@pytest.mark.parametrize("name", ["ffma-v0-local", "tc-compact", "stream-256"])
def test_nan_component_stays_in_its_rows(name, monkeypatch):
    """The first molecule's h0 rows, message weights and d_out rows NaN: every other node's final state and d h0, and every other
    message's d w, are finite and equal the run with that molecule finite."""
    c = CASES[name]
    adj, indeg, h0 = make_batch(c.batch, c.D, c.T)
    _, tgt, _ = O.message_arrays(adj)
    first = np.zeros(indeg.shape[0], bool)
    first[:5] = True   # molecule 0 owns nodes 0 .. at least 4; grow it to its whole component
    changed = True
    while changed:
        changed = False
        for a in adj:
            hit = first[a[:, 0]] | first[a[:, 1]]
            new = first.copy()
            new[a[hit].ravel()] = True
            changed |= bool((new != first).any())
            first = new
    poison_msg = first[tgt]
    results = []
    for poisoned in (False, True):
        h = h0.copy()
        M = sum(a.shape[0] for a in adj)
        mw = draw_weights(M, "signed")
        g_out = np.random.default_rng(12).normal(size=h0.shape).astype(np.float32)
        if poisoned:
            h[first] = np.nan
            mw[poison_msg] = np.nan
            g_out[first] = np.nan
        r = Run(c, monkeypatch, save=True, det=True, batch=(adj, indeg, h), mw=mw)
        out = r.forward()
        dmw, dh0, _ = r.backward(g_out)
        results.append((out[~first], dh0[~first], dmw[~poison_msg]))
    for a, b, what in zip(results[0], results[1], ("state", "d h0", "d w")):
        assert np.all(np.isfinite(b)), what
        if c.precision == "fp32":
            np.testing.assert_array_equal(b, a, err_msg=what)
        else:
            assert U.max_rel_err(b, a) < 1e-6, (what, U.max_rel_err(b, a))


# ---------------------------------------------------------------------------------------------------------------- end to end
def test_learned_edge_gate_end_to_end(monkeypatch):
    """theta [F] scores every message from its features f [M, F]; w = sigmoid(f . theta) weighs the messages through
    ``chem_sparse.propagate``, then a gated readout per graph and a squared loss.  theta's gradient (and h0's) against float64 autograd."""
    import torch
    from gated_graph_neural_network_samples_b200.chem_sparse import propagate
    c = CASES["tc-compact"]
    _env(monkeypatch, {})
    _, b = U.molecule_batch(12, c.D, c.T, 0)
    adj = [np.asarray(a, np.int32).reshape(-1, 2) for a in b["adjacency_lists"]]
    indeg = _indeg(adj, b["initial_node_representation"].shape[0], c.T)
    h0 = b["initial_node_representation"].astype(np.float32)
    gnl = np.asarray(b["graph_nodes_list"], np.int64)
    G = int(gnl.max()) + 1
    M = sum(a.shape[0] for a in adj)
    rng = np.random.default_rng(13)
    F = 6
    feats = rng.normal(size=(M, F)).astype(np.float32)
    theta0 = rng.normal(0, 0.5, F).astype(np.float32)
    w = layer_weights(c)
    rg, rt = rng.normal(0, 0.1, (2 * c.D, 1)).astype(np.float32), rng.normal(0, 0.1, (c.D, 1)).astype(np.float32)
    target = rng.normal(size=G).astype(np.float32)

    def loss_of(theta, h0t, prop, dev, dtype):
        mw = torch.sigmoid(torch.tensor(feats, dtype=dtype, device=dev) @ theta)
        out = prop(h0t, mw)
        gate = torch.sigmoid(torch.cat([out, h0t], -1) @ torch.tensor(rg, dtype=dtype, device=dev))
        val = gate * (out @ torch.tensor(rt, dtype=dtype, device=dev))
        pred = torch.zeros(G, 1, dtype=dtype, device=dev).index_add(0, torch.tensor(gnl, device=dev), val).squeeze(-1)
        return ((pred - torch.tensor(target, dtype=dtype, device=dev)) ** 2).sum()

    eng = engine_for(c)
    eng.set_graph_prepared(eng.prepare_graph_sparse_weighted(adj, indeg, save_for_backward=True))
    layers = [{k: v.detach().clone().requires_grad_(True) for k, v in lw.items()} for lw in U.to_cuda_weights(w)]
    theta = torch.tensor(theta0, device="cuda", requires_grad=True)
    th0 = torch.tensor(h0, device="cuda", requires_grad=True)
    loss = loss_of(theta, th0, lambda h, mw: propagate(eng, h, layers, mw), "cuda", torch.float32)
    loss.backward()
    rtheta = torch.tensor(theta0, dtype=torch.float64, requires_grad=True)
    rh0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    rlayers = [{k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in lw.items()} for lw in w]
    rloss = loss_of(rtheta, rh0, lambda h, mw: MW.propagation_torch(h, adj, indeg, rlayers, params(c), mw, dtype=torch.float64), "cpu",
                    torch.float64)
    rloss.backward()
    assert abs(float(loss) - float(rloss)) <= 1e-4 * abs(float(rloss)) + 1e-6
    assert U.max_rel_err(theta.grad.cpu().numpy(), rtheta.grad.numpy()) < GRAD_BAR
    assert U.max_rel_err(th0.grad.cpu().numpy(), rh0.grad.numpy()) < GRAD_BAR
    for l, lw in enumerate(rlayers):
        for k, t in lw.items():
            assert U.max_rel_err(layers[l][k].grad.cpu().numpy(), t.grad.numpy()) < GRAD_BAR, k
