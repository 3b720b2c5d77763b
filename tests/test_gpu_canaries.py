"""GPU: memory canaries.  Every other test feeds finite data into buffers that hold exactly what the call needs, so a read of another
component's row, of a caller buffer's neighbour or of an earlier batch's workspace is multiplied by zero or lands in a discarded row, and a
store past an output's end lands in memory nobody compares.  Here NaNs stand in for that memory, so such a read or store shows up:

A. Isolation.  Whole connected components (dense model: whole graphs) get a payload NaN in every ``h0`` row and in ``d_out``.  The clean
   components' final state, every ``node_states_per_layer`` entry and ``d h0`` must keep the clean run's bits and stay NaN-free.  (The
   forward has no atomics; the tile-local and GLOBAL wgmma plans are held to the rule of tests/test_gpu_engine_lifetime.py, bits or
   TILE_LOCAL_NOISE, as their MMA issue order is not fixed.)  With the poisoned components' ``h0`` finite at 100x scale and their
   ``d_out`` zero instead, every intermediate of theirs is an exact zero in the backward: in deterministic mode two draws give the same
   weight-gradient bits, and those match float64 autograd of the batch with those rows of ``d_out`` zero.  The readout keeps the clean
   graphs' bits on its grouped, permuted and dense-masked variants (the atomic one within its bar).
B. Guard bands.  Every device pointer a call takes sits between two bands of payload NaN (``guarded``); written-only outputs start as
   payload NaN, accumulators as a finite prefill.  Results must equal the same call on plain buffers, hold no payload word, and leave both
   bands intact -- at node counts and hidden sizes that put every kernel's last tile at an awkward row.
C. Leftovers.  One engine runs a clean batch, a larger all-NaN batch, a forward with NaN weights (bound, then restored in place and bound
   again, as the plug-ins do after Adam), the clean batch again (its bits) and a smaller batch (a fresh engine's result).  The NaN batch
   also leaves NaN in the SMs' shared memory for the next launch's blocks most of the time -- the one test where stale shared memory
   holds NaN, though not every time; it is not repeated to chase that.
D. Aliasing.  ``ggnn_forward`` refuses ``h_out`` overlapping ``h0`` on every model and plan, before any launch and with the engine's state
   untouched; ``d_h0`` may alias ``d_h_out`` in both backward calls and gives the out-of-place bits.

The case tables and the plan pins without a GPU are in tests/test_canaries_cpu.py.
"""
import numpy as np
import pytest

from gated_graph_neural_network_samples_b200.engine import GCNEngine, GgnnError, PropagationEngine
from oracle import ggnn_oracle as O
from tests import gcn_oracle as G
from tests import test_canaries_cpu as K
from tests.test_backward_plans_cpu import (DENSE_CASES, DENSE_STEPS, DENSE_T, FFMA_GLOBAL, GCN_CASES, GCN_FFMA, GCN_LAYERS, GCN_TC_GLOBAL,
                                           GCN_TC_LOCAL, SPARSE_CASES, dense_params, gcn_batch, plan_matches, sparse_batch)
from tests.test_gpu_backward import _autograd_reference, _cmp
from tests.test_gpu_backward_plans import _weights
from tests.test_gpu_engine_lifetime import _same

pytestmark = pytest.mark.gpu

REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}
DROP_SEED = 4242
GCN_GRAD_BAR = 2.5e-5


def _env(monkeypatch, env):
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM", "GGNN_FFMA_VARIANT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _np(ts):
    return [{k: v.cpu().numpy() for k, v in d.items()} for d in ts]


# ---------------------------------------------------------------------------------------------------------------- runners
class Ggnn:
    """One GGNN engine with save_for_backward on, its weights bound and its graph set (sparse lists or a dense matrix)."""

    def __init__(self, params, T, w_np, precision, graph, keep=1.0, det=True):
        self.eng = PropagationEngine(params, T, precision=precision)
        self.dev_w = [{REN.get(k, k): _cuda(v) for k, v in lw.items()} for lw in w_np]
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(True)
        self.eng.set_deterministic(det)
        if keep < 1.0:
            self.eng.set_state_dropout(keep, DROP_SEED)
        self.set_graph(graph)

    def set_graph(self, graph):
        if isinstance(graph, np.ndarray):
            self.eng.set_graph_dense(graph)
        else:
            self.eng.set_graph_sparse(*graph)

    def run(self, h0, g):
        import torch
        eng = self.eng
        th0 = _cuda(h0)
        self.keep_states = (th0, eng.forward(th0))   # node_states_per_layer[0] and [L]: the backward reads them again
        states = [eng.layer_state(l).cpu().numpy() for l in range(eng.L + 1)]
        grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in self.dev_w]
        dh0 = torch.zeros_like(th0)
        eng.backward(_cuda(g), grads, dh0)
        eng.sync_check()
        return {"states": states, "dh0": dh0.cpu().numpy(), "grads": _np(grads)}


class Gcn:
    def __init__(self, D, L, V, lst, w, ks, bs, precision, keep=1.0, det=True):
        self.eng = GCNEngine(D, L, use_bias=True, precision=precision)
        self.dk, self.db = [_cuda(k) for k in ks], [_cuda(b) for b in bs]
        self.eng.set_weights(self.dk, self.db)
        self.eng.set_save_for_backward(True)
        self.eng.set_deterministic(det)
        self.eng.set_state_dropout(keep, DROP_SEED)
        self.eng.set_graph_gcn(V, lst, w)
        self.keep = keep

    def run(self, h0, g):
        import torch
        eng = self.eng
        th0 = _cuda(h0)
        self.keep_states = (th0, eng.forward(th0))   # node_states_per_layer[0] and [L]: the backward reads them again
        states = [eng.layer_state(l).cpu().numpy() for l in range(eng.L + 1)]
        grads = [{"kernel": torch.zeros_like(k), "bias": torch.zeros_like(b)} for k, b in zip(self.dk, self.db)]
        dh0 = torch.zeros_like(th0)
        eng.backward(_cuda(g), grads, dh0)
        eng.sync_check()
        return {"states": states, "dh0": dh0.cpu().numpy(), "grads": _np(grads)}


# ---------------------------------------------------------------------------------------------------------------- A. isolation
def _isolation(tag, runner, bad, h0, g, reference, compare):
    """``bad``: boolean row mask of the poisoned components.  ``reference(h0, g)`` -> float64 (out, d h0, [per-layer grads keyed as the
    engine's]) of the whole batch; ``compare(got, ref, tag)`` asserts one gradient against it at the model's bar.  The forward is held to
    bits on every plan: two runs on one engine repeat theirs, the wgmma plans included (their MMA issue order varies only between
    engines, which is where tests/test_gpu_engine_lifetime.py allows TILE_LOCAL_NOISE)."""
    ok = ~bad
    clean = runner.run(h0, g)
    hp, gp = h0.copy(), g.copy()
    hp[bad], gp[bad] = K.payload_nan(hp[bad].shape), K.payload_nan(gp[bad].shape)
    pois = runner.run(hp, gp)
    for l, (a, b) in enumerate(zip(clean["states"], pois["states"])):
        assert np.all(np.isfinite(b[ok])), (tag, "NaN in clean rows of layer state", l)
        np.testing.assert_array_equal(b[ok], a[ok], err_msg="%s layer state %d" % (tag, l))
    assert np.all(np.isfinite(pois["dh0"][ok])), (tag, "NaN in clean rows of d h0")
    np.testing.assert_array_equal(pois["dh0"][ok], clean["dh0"][ok], err_msg=tag + " d h0")
    # weight gradients: the poisoned components finite at 100x, their d_out zero -> every intermediate of theirs is an exact zero
    g0 = g.copy()
    g0[bad] = 0.0
    draws = []
    for seed in (1, 2):
        hs = h0.copy()
        hs[bad] = 100.0 * np.random.default_rng(seed).normal(0, 1, hs[bad].shape).astype(np.float32)
        draws.append((hs, runner.run(hs, g0)))
    (h1, r1), (_, r2) = draws
    for l, (a, b) in enumerate(zip(r1["grads"], r2["grads"])):
        for k in a:
            assert np.all(np.isfinite(a[k])), (tag, l, k)
            np.testing.assert_array_equal(a[k], b[k], err_msg="%s layer %d %s: two draws of the poisoned components" % (tag, l, k))
    np.testing.assert_array_equal(r1["dh0"][ok], r2["dh0"][ok], err_msg=tag)
    np.testing.assert_array_equal(r1["states"][-1][ok], clean["states"][-1][ok], err_msg=tag + " forward beside 100x components")
    ref_out, ref_dh0, ref_gw = reference(h1, g0)
    compare(r1["dh0"][ok], ref_dh0[ok], tag + " d h0 (clean rows)")
    for l, (a, r) in enumerate(zip(r1["grads"], ref_gw)):
        for k in r:
            compare(a[k].reshape(r[k].shape), r[k], "%s layer %d %s" % (tag, l, k))


def _gcn_cmp(got, ref, tag):
    err = _rel_err(got, ref)
    print("grad %-28s max|err|/max|ref| = %.2e" % (tag, err))
    assert err < GCN_GRAD_BAR, (tag, err)


def _rel_err(a, b):
    s = max(float(np.max(np.abs(b))), 1e-12)
    return float(np.max(np.abs(a - b))) / s


def _ggnn_reference(params, T, w, adj, indeg, keep):
    drop = (keep, DROP_SEED) if keep < 1.0 else None

    def ref(h0, g):
        out, dh0, gw = _autograd_reference(params, T, w, adj, indeg, h0, g, state_dropout=drop)
        return out, dh0, [{REN.get(k, k): v for k, v in lw.items()} for lw in gw]
    return ref


@pytest.mark.parametrize("name", sorted(K.ISOLATION_SPARSE_BY_NAME))
def test_poisoned_components_do_not_reach_clean_ones_sparse(name, monkeypatch):
    c, keep = K.ISOLATION_SPARSE_BY_NAME[name]
    _env(monkeypatch, c.env)
    adj, indeg, h0 = sparse_batch(c.batch, c.params["hidden_size"], c.T)
    w = _weights(c.params, c.T)
    g = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    r = Ggnn(c.params, c.T, w, c.precision, (adj, indeg), keep=keep)
    assert plan_matches(r.eng.plan, c.plan), (c.plan, r.eng.plan)
    labels, bad_ids = K.sparse_isolation_batch(c, r.eng.prepare_graph_sparse(adj, indeg).arrays(c.T)["tile_start"])[3:]
    _isolation(name, r, np.isin(labels, bad_ids), h0, g, _ggnn_reference(c.params, c.T, w, adj, indeg, keep), _cmp)


@pytest.mark.parametrize("name,precision,D,weighted,pattern", DENSE_CASES, ids=[c[0] for c in DENSE_CASES])
def test_poisoned_graphs_do_not_reach_clean_ones_dense(name, precision, D, weighted, pattern):
    import torch
    A, h0, bad_graphs = K.dense_isolation_batch(D, weighted)
    b, v = h0.shape[:2]
    dw = O.init_dense_weights({"hidden_size": D}, DENSE_T, np.random.default_rng(5))
    dw["cand_bias"] = np.random.default_rng(6).normal(0, 0.1, D).astype(np.float32)
    w_eng = [dict(dw, edge_biases=dw["edge_biases"].reshape(DENSE_T, D))]
    r = Ggnn(dense_params(D), DENSE_T, w_eng, precision, A)
    assert plan_matches(r.eng.plan, pattern), (pattern, r.eng.plan)

    def ref(h, g):
        tw = {k: torch.tensor(x, dtype=torch.float64, requires_grad=True) for k, x in dw.items()}
        th = torch.tensor(h.reshape(b, v, D), dtype=torch.float64, requires_grad=True)
        out = O.dense_propagation_torch(th, A, tw, {"num_timesteps": DENSE_STEPS, "use_edge_bias": True}, dtype=torch.float64)
        (out * torch.tensor(g.reshape(b, v, D), dtype=torch.float64)).sum().backward()
        return out.detach().numpy().reshape(b * v, D), th.grad.numpy().reshape(b * v, D), [{k: tw[k].grad.numpy() for k in tw}]

    g = np.random.default_rng(7).normal(size=(b * v, D)).astype(np.float32)
    bad = np.repeat(np.isin(np.arange(b), bad_graphs), v)
    _isolation("dense " + name, r, bad, h0.reshape(b * v, D).copy(), g, ref, _cmp)


@pytest.mark.parametrize("name,precision,D,kind,keep,env,pattern", GCN_CASES, ids=[c[0] for c in GCN_CASES])
def test_poisoned_components_do_not_reach_clean_ones_gcn(name, precision, D, kind, keep, env, pattern, monkeypatch):
    import torch
    _env(monkeypatch, env)
    V, lst, w, ks, bs, h0 = K.gcn_isolation_batch(D, kind)[:6]
    g = np.random.default_rng(5).normal(0, 1, (V, D)).astype(np.float32)
    r = Gcn(D, GCN_LAYERS, V, lst, w, ks, bs, precision, keep=keep)
    assert plan_matches(r.eng.plan, pattern), (pattern, r.eng.plan)
    labels, runs = K.gcn_isolation_batch(D, kind, r.eng.prepare_graph_gcn(V, lst, w).arrays(1)["tile_start"])[6:]
    masks = [r.eng.state_dropout_mask(l, keep, DROP_SEED) for l in range(GCN_LAYERS - 1)] if keep < 1 else None

    def ref(h, gg):
        th = torch.from_numpy(h).double().requires_grad_()
        tk = [torch.from_numpy(k).double().requires_grad_() for k in ks]
        tb = [torch.from_numpy(x).double().requires_grad_() for x in bs]
        out = G.gcn_propagation_torch(th, lst, torch.from_numpy(w).double(), tk, tb, masks, keep)
        out.backward(torch.from_numpy(gg).double())
        return out.detach().numpy(), th.grad.numpy(), [{"kernel": a.grad.numpy(), "bias": b.grad.numpy()} for a, b in zip(tk, tb)]

    for i, bad_ids in enumerate(runs):
        _isolation("gcn %s run %d" % (name, i), r, np.isin(labels, bad_ids), h0, g, ref, _gcn_cmp)


def _readout_ws(D, seed=3):
    rng = np.random.default_rng(seed)
    return [_cuda(rng.normal(0, 0.3, n)) for n in (2 * D, 1, D, 1)]


@pytest.mark.parametrize("variant", ["grouped", "permuted", "atomic", "dense-masked"])
def test_readout_keeps_clean_graphs_beside_nan_graphs(variant):
    """The readout sums each graph's rows; NaN rows of other graphs (h_last, h0 and their d_out) must not reach a clean graph's ``out`` or
    its rows of ``d_h_last``.  Grouped, permuted under deterministic mode and dense-masked: bits; atomic: within 1e-6, NaN-free."""
    D, Gn = 36, 300
    rng = np.random.default_rng(11)
    eng = PropagationEngine({"hidden_size": D, "layer_timesteps": [1], "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}, 2)
    if variant == "dense-masked":
        v = 9
        gnl = np.repeat(np.arange(Gn, dtype=np.int32), v)
        mask = (rng.random((Gn, v)) < 0.7).astype(np.float32)
        eng.readout_set_graphs(Gn, nodes_per_graph=v, node_mask=mask)
    else:
        sizes = rng.integers(0, 12, Gn)
        gnl = np.repeat(np.arange(Gn, dtype=np.int32), sizes)
        if variant != "grouped":
            gnl = rng.permutation(gnl)
        eng.set_deterministic(variant == "permuted")
        eng.readout_set_graphs(Gn, graph_nodes_list=gnl)
    V = gnl.shape[0]
    h, h0 = rng.normal(0, 0.5, (V, D)).astype(np.float32), rng.normal(0, 0.5, (V, D)).astype(np.float32)
    d_out = rng.normal(size=Gn).astype(np.float32)
    bad_g = K.poisoned_components(Gn)
    bad = np.isin(gnl, bad_g)
    ws = _readout_ws(D)

    def run(hh, hh0, dd):
        out = eng.readout_forward(_cuda(hh), _cuda(hh0), *ws)
        d_h = eng.readout_backward(_cuda(hh), _cuda(hh0), *ws, _cuda(dd))[0]
        eng.sync_check()
        return out.cpu().numpy(), d_h.cpu().numpy()

    o1, d1 = run(h, h0, d_out)
    hp, h0p, dp = h.copy(), h0.copy(), d_out.copy()
    hp[bad], h0p[bad], dp[bad_g] = K.payload_nan(1)[0], np.nan, np.nan
    o2, d2 = run(hp, h0p, dp)
    okg = ~np.isin(np.arange(Gn), bad_g)
    assert np.all(np.isfinite(o2[okg])) and np.all(np.isfinite(d2[~bad]))
    if variant == "atomic":
        assert _rel_err(o2[okg], o1[okg]) < 1e-6
    else:
        np.testing.assert_array_equal(o2[okg], o1[okg])
    np.testing.assert_array_equal(d2[~bad], d1[~bad])


# ---------------------------------------------------------------------------------------------------------------- B. guard bands
def _g(shape, fill=None):
    """A guarded fp32 CUDA view of ``shape``; ``fill``: None keeps the payload NaN (written-only outputs), else the values copied in."""
    n = int(np.prod(shape))
    gb = K.guarded(n)
    if fill is not None:
        gb.view.copy_(_cuda(np.asarray(fill, np.float32).reshape(-1)))
    gb.t = gb.view.view(*shape)
    return gb


@pytest.mark.parametrize("shape", K.GUARD_SHAPES, ids=[s[0] for s in K.GUARD_SHAPES])
def test_guard_bands_around_every_ggnn_buffer(shape, monkeypatch):
    """Forward with save and backward with every caller pointer guarded (h0, h_out, every weight, d_out, d h0, every gradient prefilled),
    against the same calls on plain buffers: the same bits, no payload word in an output, every band intact."""
    import torch
    name, V, D, precision, env, pattern = shape
    _env(monkeypatch, env)
    T = 4
    p = K.guard_params(D)
    adj, indeg = K.chain_batch(V)
    w = _weights(p, T)
    rng = np.random.default_rng(9)
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    g = rng.normal(0, 1, (V, D)).astype(np.float32)
    pre = [{REN.get(k, k): rng.normal(0, 1, v.shape).astype(np.float32) for k, v in lw.items()} for lw in w]

    def run(guard):
        eng = PropagationEngine(p, T, precision=precision)
        eng.set_deterministic(True)
        mk = (lambda s, f=None: _g(s, f)) if guard else None
        keep = []

        def buf(s, f=None):
            if guard:
                b = mk(s, f)
                keep.append(b)
                return b.t
            return (_cuda(f) if f is not None else torch.empty(s, device="cuda")).reshape(s)
        dev_w = [{REN.get(k, k): buf(v.shape, v) for k, v in lw.items()} for lw in w]
        eng.set_weights(dev_w)
        eng.set_save_for_backward(True)
        eng.set_graph_sparse(adj, indeg)
        assert plan_matches(eng.plan, pattern), (pattern, eng.plan)
        th0, out = buf((V, D), h0), buf((V, D))
        eng.forward(th0, out)
        grads = [{k: buf(v.shape, v) for k, v in lw.items()} for lw in pre]
        dh0 = buf((V, D))
        eng.backward(buf((V, D), g), grads, dh0)
        eng.sync_check()
        outs = [out, dh0] + [t for lw in grads for t in lw.values()]
        if guard:
            assert not any(K.has_payload(t) for t in outs), name
            assert all(b.bands_intact() for b in keep), name
        return [t.cpu().numpy() for t in outs]

    for a, b in zip(run(True), run(False)):
        np.testing.assert_array_equal(a, b, err_msg=name)


@pytest.mark.parametrize("D,V", [(12, 17), (100, 129), (256, 65)])
def test_guard_bands_around_every_gcn_buffer(D, V):
    import torch
    L = 2
    rng = np.random.default_rng(D)
    Vc, lst, w = G.component_list([int(x) for x in np.diff(np.r_[0, np.sort(rng.choice(np.arange(1, V), 4, replace=False)), V])], rng)
    assert Vc == V
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)]
    h0, g = rng.normal(0, 1, (V, D)).astype(np.float32), rng.normal(0, 1, (V, D)).astype(np.float32)
    pk, pb = rng.normal(0, 1, (D, D)).astype(np.float32), rng.normal(0, 1, D).astype(np.float32)

    def run(guard, precision):
        keep = []

        def buf(s, f=None):
            if guard:
                b = _g(s, f)
                keep.append(b)
                return b.t
            return (_cuda(f) if f is not None else torch.empty(s, device="cuda")).reshape(s)
        eng = GCNEngine(D, L, use_bias=True, precision=precision)
        eng.set_deterministic(True)
        eng.set_weights([buf((D, D), k) for k in ks], [buf((D,), b) for b in bs])
        eng.set_save_for_backward(True)
        eng.set_graph_gcn(V, lst, w)
        th0, out = buf((V, D), h0), buf((V, D))   # both alive until the backward, which reads them again
        eng.forward(th0, out)
        grads = [{"kernel": buf((D, D), pk), "bias": buf((D,), pb)} for _ in range(L)]
        dh0 = buf((V, D))
        eng.backward(buf((V, D), g), grads, dh0)
        eng.sync_check()
        outs = [out, dh0] + [t for d in grads for t in d.values()]
        if guard:
            assert not any(K.has_payload(t) for t in outs)
            assert all(b.bands_intact() for b in keep)
        return [t.cpu().numpy() for t in outs]

    for precision in ("bf16x3", "fp32"):
        for a, b in zip(run(True, precision), run(False, precision)):
            np.testing.assert_array_equal(a, b, err_msg=precision)


class _Plain:
    """A plain CUDA buffer with the face of ``K.Guarded`` (``t``, ``bands_intact``), for the unguarded twin of a guarded call."""

    def __init__(self, shape, fill=None):
        import torch
        self.t = _cuda(fill).reshape(shape) if fill is not None else torch.empty(shape, device="cuda")

    def bands_intact(self):
        return True


@pytest.mark.parametrize("Gn", [1, 300])
def test_guard_bands_around_the_readout_and_the_fused_loss(Gn):
    """The readout's seven (forward) and thirteen (backward) pointers guarded, one graph and more than 256; the fused loss with its
    readout trainables guarded."""
    D = 36
    rng = np.random.default_rng(Gn)
    gnl = np.repeat(np.arange(Gn, dtype=np.int32), rng.integers(1, 9, Gn))
    V = gnl.shape[0]
    h, h0 = rng.normal(0, 0.5, (V, D)).astype(np.float32), rng.normal(0, 0.5, (V, D)).astype(np.float32)
    wv = [rng.normal(0, 0.3, n).astype(np.float32) for n in (2 * D, 1, D, 1)]
    d_out = rng.normal(size=Gn).astype(np.float32)
    pre = [rng.normal(0, 1, n).astype(np.float32) for n in (2 * D, 1, D, 1)]
    eng = PropagationEngine({"hidden_size": D, "layer_timesteps": [1], "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}, 2)
    eng.set_deterministic(True)
    eng.readout_set_graphs(Gn, graph_nodes_list=gnl)
    res = {}
    for guard in (True, False):
        mk = _g if guard else _Plain
        ins = [mk((V, D), h), mk((V, D), h0)] + [mk(x.shape, x) for x in wv]
        out, dd, dh = mk((Gn,)), mk((Gn,), d_out), mk((V, D))
        gw = [mk(x.shape, x) for x in pre]
        ptr = lambda b: b.t.data_ptr()
        eng._check(eng.lib.ggnn_readout_forward(eng._h, *[ptr(b) for b in ins], ptr(out), eng._stream()))
        eng._check(eng.lib.ggnn_readout_backward(eng._h, *[ptr(b) for b in ins], ptr(dd), ptr(dh), *[ptr(b) for b in gw], eng._stream()))
        eng.sync_check()
        outs = [out.t, dh.t] + [b.t for b in gw]
        assert not (guard and any(K.has_payload(t) for t in outs))
        assert all(b.bands_intact() for b in ins + [out, dd, dh] + gw)
        res[guard] = [t.cpu().numpy() for t in outs]
    for a, b in zip(res[True], res[False]):
        np.testing.assert_array_equal(a, b)
    # the fused loss: a batch without edges through one GRU step, the readout trainables guarded
    adj = [np.zeros((0, 2), np.int32)] * 2
    indeg = np.zeros((V, 2), np.float32)
    eng.set_weights([{"edge_weights": _cuda(rng.normal(0, 0.1, (2, D, D))), "gate_kernel": _cuda(rng.normal(0, 0.1, (2 * D, 2 * D))),
                      "gate_bias": _cuda(np.zeros(2 * D)), "cand_kernel": _cuda(rng.normal(0, 0.1, (2 * D, D))), "cand_bias": _cuda(np.zeros(D))}])
    tv, tm = rng.normal(size=(1, Gn)).astype(np.float32), np.ones((1, Gn), np.float32)
    fused = {}
    for guard in (True, False):
        bs = [(_g if guard else _Plain)(x.shape, x) for x in wv]
        fused[guard] = eng.run_sparse_host_readout(adj, indeg, h0, gnl, Gn, [tuple(b.t for b in bs)], tv, tm)
        assert all(b.bands_intact() for b in bs)
    for a, b in zip(fused[True], fused[False]):
        np.testing.assert_array_equal(a, b)


def test_guard_bands_around_the_dataset_outputs():
    """``ggnn_set_graph_dataset`` and ``ggnn_set_graph_dataset_dense`` write h0, the targets, the target mask (and the node mask) into the
    caller's buffers: through guarded pointers they write the same values, no payload word and nothing outside."""
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset
    from tests.test_dense_device_data_cpu import edge_types, flat_of, molecules, params
    from tests.test_device_data_cpu import GRU, T, sparse_graph_set
    sets = []
    eng = PropagationEngine(dict(GRU, hidden_size=36), T, precision="bf16x3")
    sets.append((eng, DeviceDataset.for_engine(eng, packing.FlatSparseGraphs(sparse_graph_set(), T)), [np.arange(17), np.array([3])], None))
    deng = PropagationEngine(params(20), edge_types(True), precision="fp32")
    v = int(max(packing.DEFAULT_BUCKET_SIZES))
    sets.append((deng, DeviceDataset.for_engine(deng, flat_of(molecules(), True)), [np.arange(0, 40, 3), np.array([5])], v))
    for e, ds, batches, v in sets:
        for ids in batches:
            b = ds.prepare_batch(ids, save_for_backward=True, nodes_per_graph=v)
            want = [t.cpu().numpy() for t in e.set_graph_from_dataset(b)]
            shapes = [(b.V, e.D), (ds.num_tasks, b.G), (ds.num_tasks, b.G)] + ([(b.G * v,)] if v else [])
            gb = [_g(s) for s in shapes]
            fn = e.lib.ggnn_set_graph_dataset_dense if v else e.lib.ggnn_set_graph_dataset
            e._check(fn(e._h, b._h, *[x.t.data_ptr() for x in gb], e._stream()))
            e.sync_check()
            for x, wv in zip(gb, want):
                assert not K.has_payload(x.t) and x.bands_intact()
                np.testing.assert_array_equal(x.t.cpu().numpy().reshape(wv.shape), wv)


# ---------------------------------------------------------------------------------------------------------------- C. leftovers
@pytest.mark.parametrize("name", K.LEFTOVER_FAMILIES)
def test_one_engine_forgets_a_nan_batch_and_nan_weights(name, monkeypatch):
    c = SPARSE_CASES[name]
    _env(monkeypatch, c.env)
    D = c.params["hidden_size"]
    w = _weights(c.params, c.T)
    bat = {t: sparse_batch(kind, D, c.T) for t, kind in K.LEFTOVER_BATCHES.items()}
    gA = np.random.default_rng(5).normal(size=bat["A"][2].shape).astype(np.float32)
    r = Ggnn(c.params, c.T, w, c.precision, bat["A"][:2])
    assert plan_matches(r.eng.plan, c.plan), (c.plan, r.eng.plan)
    first = r.run(bat["A"][2], gA)
    plan = r.eng.plan
    # a larger batch, all NaN
    P = bat["P"]
    r.set_graph(P[:2])
    nan_p = K.payload_nan(P[2].shape)
    nanrun = r.run(nan_p, nan_p)
    assert nanrun["states"][-1].shape == P[2].shape
    # NaN weights bound, a forward on P, then the values restored in place and bound again
    saved = [{k: v.clone() for k, v in lw.items()} for lw in r.dev_w]
    for lw in r.dev_w:
        for v in lw.values():
            v.fill_(float("nan"))
    r.eng.set_weights(r.dev_w)
    r.eng.forward(_cuda(P[2]))
    r.eng.sync_check()
    for lw, sv in zip(r.dev_w, saved):
        for k in lw:
            lw[k].copy_(sv[k])
    r.eng.set_weights(r.dev_w)
    # A again: its bits
    r.set_graph(bat["A"][:2])
    again = r.run(bat["A"][2], gA)
    assert r.eng.plan == plan
    for l, (a, b) in enumerate(zip(first["states"], again["states"])):
        np.testing.assert_array_equal(b, a, err_msg="%s A again layer %d" % (name, l))
    np.testing.assert_array_equal(again["dh0"], first["dh0"])
    for l, (a, b) in enumerate(zip(first["grads"], again["grads"])):
        for k in a:
            np.testing.assert_array_equal(b[k], a[k], err_msg="%s A again layer %d %s" % (name, l, k))
    # a smaller batch: a fresh engine's result, NaN-free
    B = bat["B"]
    gB = np.random.default_rng(6).normal(size=B[2].shape).astype(np.float32)
    r.set_graph(B[:2])
    small = r.run(B[2], gB)
    fresh = Ggnn(c.params, c.T, w, c.precision, B[:2]).run(B[2], gB)
    for l, (a, b) in enumerate(zip(fresh["states"], small["states"])):
        assert np.all(np.isfinite(b))
        _same(b, a, plan, "%s B layer %d" % (name, l))
    np.testing.assert_array_equal(small["dh0"], fresh["dh0"])
    for l, (a, b) in enumerate(zip(fresh["grads"], small["grads"])):
        for k in a:
            assert np.all(np.isfinite(b[k]))
            np.testing.assert_array_equal(b[k], a[k], err_msg="%s B layer %d %s" % (name, l, k))
    # the readout map: a NaN readout between two clean ones
    gnl = np.repeat(np.arange(24, dtype=np.int32), np.diff(np.linspace(0, B[2].shape[0], 25).astype(int)))
    ws = _readout_ws(D)
    hB = _cuda(small["states"][-1])
    r.eng.readout_set_graphs(24, graph_nodes_list=gnl)
    ro1 = r.eng.readout_forward(hB, _cuda(B[2]), *ws).cpu().numpy()
    nanP = _cuda(nan_p)
    r.eng.readout_set_graphs(5, graph_nodes_list=np.sort(np.random.default_rng(1).integers(0, 5, P[2].shape[0])).astype(np.int32))
    r.eng.readout_forward(nanP, nanP, *ws)
    r.eng.readout_set_graphs(24, graph_nodes_list=gnl)
    ro2 = r.eng.readout_forward(hB, _cuda(B[2]), *ws).cpu().numpy()
    np.testing.assert_array_equal(ro2, ro1)
    assert np.all(np.isfinite(ro2))


GCN_PLANS = [("bf16x3", 100, "components", GCN_TC_LOCAL), ("bf16x3", 128, "random", GCN_TC_GLOBAL), ("fp32", 132, "components", GCN_FFMA)]


@pytest.mark.parametrize("precision,D,kind,pattern", GCN_PLANS, ids=["local", "global", "fp32"])
def test_one_gcn_engine_forgets_a_nan_batch_and_nan_weights(precision, D, kind, pattern, monkeypatch):
    _env(monkeypatch, {})
    V, lst, w, ks, bs, h0 = gcn_batch(D, kind)
    g = np.random.default_rng(5).normal(0, 1, (V, D)).astype(np.float32)
    r = Gcn(D, GCN_LAYERS, V, lst, w, ks, bs, precision)
    assert plan_matches(r.eng.plan, pattern), (pattern, r.eng.plan)
    first = r.run(h0, g)
    plan = r.eng.plan
    rng = np.random.default_rng(2)
    VP = 2 * V + 50
    lp, wp = G.random_gcn_list(VP, 8 * VP, rng)
    r.eng.set_graph_gcn(VP, lp, wp)
    nan_p = K.payload_nan((VP, D))
    r.run(nan_p, nan_p)
    saved = [t.clone() for t in r.dk + r.db]
    for t in r.dk + r.db:
        t.fill_(float("nan"))
    r.eng.set_weights(r.dk, r.db)
    r.eng.forward(_cuda(rng.normal(0, 1, (VP, D))))
    r.eng.sync_check()
    for t, s in zip(r.dk + r.db, saved):
        t.copy_(s)
    r.eng.set_weights(r.dk, r.db)
    r.eng.set_graph_gcn(V, lst, w)
    again = r.run(h0, g)
    assert r.eng.plan == plan
    for a, b in zip(first["states"], again["states"]):
        np.testing.assert_array_equal(b, a)
    np.testing.assert_array_equal(again["dh0"], first["dh0"])
    for a, b in zip(first["grads"], again["grads"]):
        for k in a:
            np.testing.assert_array_equal(b[k], a[k])
    VB = V // 3
    keep = np.flatnonzero((lst[:, 0] < VB) & (lst[:, 1] < VB))
    hB, gB = h0[:VB].copy(), g[:VB].copy()
    r.eng.set_graph_gcn(VB, lst[keep], w[keep])
    small = r.run(hB, gB)
    fresh = Gcn(D, GCN_LAYERS, VB, lst[keep], w[keep], ks, bs, precision).run(hB, gB)
    for a, b in zip(fresh["states"], small["states"]):
        assert np.all(np.isfinite(b))
        np.testing.assert_array_equal(b, a)
    np.testing.assert_array_equal(small["dh0"], fresh["dh0"])
    for a, b in zip(fresh["grads"], small["grads"]):
        for k in a:
            np.testing.assert_array_equal(b[k], a[k])


# ---------------------------------------------------------------------------------------------------------------- D. aliasing
ALIAS_FAMILIES = ["ffma0-local-gru-D36", "ffma-global-rnn-D100", "tc-local64-gru-D20", "tc-global-rnn-D20", "stream-forced-gru-D20",
                  "stream-rnn-D132", "ffma-local-cudnn-D100", "ffma-global-attention-D36"]


def _check_refused(eng, h0, V, D):
    """``h_out == h0`` and ``h_out = h0 + D`` are refused with GGNN_EINVAL naming both pointers; the last forward stays readable."""
    import torch
    before = eng.layer_state(eng.L).cpu().numpy()
    buf = torch.empty((V + 1) * D, device="cuda")
    buf[:V * D].copy_(h0.reshape(-1))
    a = buf[:V * D].view(V, D)
    for out in (a, buf[D:].view(V, D)):
        with pytest.raises(GgnnError) as ei:
            eng.forward(a, out)
        assert ei.value.code == -1 and "%x" % a.data_ptr() in str(ei.value) and "%x" % out.data_ptr() in str(ei.value), str(ei.value)
    np.testing.assert_array_equal(buf[:V * D].view(V, D).cpu().numpy(), h0.cpu().numpy())
    np.testing.assert_array_equal(eng.layer_state(eng.L).cpu().numpy(), before)


@pytest.mark.parametrize("name", ALIAS_FAMILIES + ["steps1", "steps0"])
def test_forward_refuses_an_overlapping_output(name, monkeypatch):
    import torch
    from tests.test_backward_plans_cpu import model
    if name in ("steps1", "steps0"):
        c = SPARSE_CASES["ffma-global-gru-D100"]
        params = model("GRU", 36, layer_timesteps=(1,) if name == "steps1" else (0,), residual_connections={})
    else:
        c = SPARSE_CASES[name]
        params = c.params
    _env(monkeypatch, c.env)
    D = params["hidden_size"]
    adj, indeg, h0 = sparse_batch(c.batch, D, c.T)
    r = Ggnn(params, c.T, _weights(params, c.T), c.precision, (adj, indeg))
    assert plan_matches(r.eng.plan, c.plan), (c.plan, r.eng.plan)
    th0 = _cuda(h0)
    out = r.eng.forward(th0)
    g = torch.ones_like(out)
    _check_refused(r.eng, th0, h0.shape[0], D)
    if sum(params["layer_timesteps"]):           # the saved activations survive the refusal: the backward runs as before
        dh_a = torch.zeros_like(th0)
        grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in r.dev_w]
        r.eng.backward(g, grads, dh_a)
        ref = Ggnn(params, c.T, _weights(params, c.T), c.precision, (adj, indeg)).run(h0, g.cpu().numpy())
        np.testing.assert_array_equal(dh_a.cpu().numpy(), ref["dh0"])


@pytest.mark.parametrize("L", [1, 3])
@pytest.mark.parametrize("precision,D,kind,pattern", [("bf16x3", 12, "components", GCN_TC_LOCAL), ("bf16x3", 128, "random", GCN_TC_GLOBAL),
                                                     ("fp32", 12, "components", GCN_FFMA)], ids=["local", "global", "fp32"])
def test_gcn_forward_refuses_an_overlapping_output(precision, D, kind, pattern, L, monkeypatch):
    """At one layer (the reference's h12_l1 shape) and at three."""
    _env(monkeypatch, {})
    V, lst, w, ks, bs, h0 = gcn_batch(D, kind)
    r = Gcn(D, L, V, lst, w, ks[:L], bs[:L], precision)
    assert plan_matches(r.eng.plan, pattern), (pattern, r.eng.plan)
    th0 = _cuda(h0)
    out = r.eng.forward(th0)   # noqa: F841  (the last forward's h_out, read after the refusals)
    _check_refused(r.eng, th0, V, D)


def test_dense_forward_refuses_an_overlapping_output():
    A, h0 = K.dense_isolation_batch(24, True)[:2]
    b, v, D = h0.shape
    dw = O.init_dense_weights({"hidden_size": D}, DENSE_T, np.random.default_rng(5))
    r = Ggnn(dense_params(D), DENSE_T, [dict(dw, edge_biases=dw["edge_biases"].reshape(DENSE_T, D))], "fp32", A)
    assert plan_matches(r.eng.plan, DENSE_CASES[0][4]), r.eng.plan
    th0 = _cuda(h0.reshape(b * v, D))
    out = r.eng.forward(th0)   # noqa: F841
    _check_refused(r.eng, th0, b * v, D)


ALIAS_BACKWARD = ["ffma0-local-gru-D36", "tc-global-rnn-D20", "stream-rnn-D132", "ffma-local-cudnn-D100", "ffma-global-attention-D36",
                  "dense-weighted-fp32", "dense-binary-tc", "gcn-local-L1", "gcn-local-L3", "gcn-global-L1", "gcn-fp32-L1", "gcn-fp32-L3"]


@pytest.mark.parametrize("name", ALIAS_BACKWARD)
def test_backward_into_its_own_gradient_buffer(name, monkeypatch):
    """``d_h0 == d_h_out``, and ``d_h0 = d_h_out + D`` (a partial overlap), give the out-of-place bits of ``d h0`` and every gradient: on
    the sparse GGNN (three plan families, CudnnCompatibleGRUCell, attention), the dense model and the GCN on its three plans."""
    import torch
    if name.startswith("gcn"):
        _, plan_kind, L = name.split("-")
        L = int(L[1:])
        precision, D, kind, pattern = {p[3]: p for p in GCN_PLANS}[{"local": GCN_TC_LOCAL, "global": GCN_TC_GLOBAL, "fp32": GCN_FFMA}[plan_kind]]
        _env(monkeypatch, {})
        V, lst, w, ks, bs, h0 = gcn_batch(D, kind)
        r = Gcn(D, L, V, lst, w, ks[:L], bs[:L], precision)
    elif name.startswith("dense"):
        cname, precision, D, weighted, pattern = DENSE_CASES[0] if name == "dense-weighted-fp32" else DENSE_CASES[2]
        A, h0 = K.dense_isolation_batch(D, weighted)[:2]
        h0 = h0.reshape(-1, D)
        V = h0.shape[0]
        dw = O.init_dense_weights({"hidden_size": D}, DENSE_T, np.random.default_rng(5))
        r = Ggnn(dense_params(D), DENSE_T, [dict(dw, edge_biases=dw["edge_biases"].reshape(DENSE_T, D))], precision, A)
    else:
        c = SPARSE_CASES[name]
        _env(monkeypatch, c.env)
        D, pattern = c.params["hidden_size"], c.plan
        adj, indeg, h0 = sparse_batch(c.batch, D, c.T)
        r = Ggnn(c.params, c.T, _weights(c.params, c.T), c.precision, (adj, indeg))
        V = h0.shape[0]
    assert plan_matches(r.eng.plan, pattern), (pattern, r.eng.plan)
    g = np.random.default_rng(3).normal(size=(V, D)).astype(np.float32)
    ref = r.run(h0, g)
    grad_like = (lambda: [{"kernel": torch.zeros_like(k), "bias": torch.zeros_like(b)} for k, b in zip(r.dk, r.db)]) if name.startswith("gcn") \
        else (lambda: [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in r.dev_w])
    for shift in (0, D):
        buf = torch.zeros((V + 1) * D, device="cuda")
        d_out = buf[D - shift:D - shift + V * D].view(V, D) if shift else buf[:V * D].view(V, D)
        d_h0 = buf[D:D + V * D].view(V, D) if shift else d_out
        d_out.copy_(_cuda(g))
        grads = grad_like()
        r.eng.backward(d_out, grads, d_h0)
        r.eng.sync_check()
        np.testing.assert_array_equal(d_h0.cpu().numpy(), ref["dh0"], err_msg="%s shift %d" % (name, shift))
        for a, b in zip(_np(grads), ref["grads"]):
            for k in a:
                np.testing.assert_array_equal(a[k], b[k], err_msg="%s shift %d %s" % (name, shift, k))
