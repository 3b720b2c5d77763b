"""GPU: one timestep of the compact tile kernel (every tile <= 64 rows) against the 128-row layout and the float64 oracle.

On compact tiles with the tile's CSR slice in shared memory, ``ggnn_fwd_tc_kernel`` gathers over real rows only, one task per (row,
8-column chunk) spread over all 512 worker threads, and on the GRU cell it writes the new state without a barrier before it.  The 128-row
layout keeps the row-per-thread gather over every allocated row and the barrier.  Both sum every message and every product in the same
order, so a graph that runs on compact tiles, and the same graph with one 100-node component appended (which moves every tile onto the
128-row layout), give the same bits on the graph's rows:

* the final state and every ``layer_state(l)``, with the default number of gather tiles and with 2 and 3;
* ``d h0`` of the backward, which reads the saved activations (``agg``, ``r``, ``u``, ``c``, ``h_in``): the appended component gets a
  zero output gradient, and no row's ``d h0`` depends on another component;
* forward and gradients are within the bars of tests/test_gpu_backward.py of float64 autograd.

With state dropout the mask depends on the node count, so the appended component would change it; those cases check the default against
two and three gather tiles bit for bit, and the forward against the oracle with the engine's mask.

Graphs: components of 1 to 64 nodes (rows not a multiple of 16), isolated nodes, self-loops, a row receiving many repeated messages of
one type, 1, 4 and 16 edge types with tiles that hold only some of them, edge bias with avg aggregation, GRU and RNN, NH 8 to 64.
"""
import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests.test_backward_plans_cpu import model
from tests.test_gpu_backward import _autograd_reference, _cmp

pytestmark = pytest.mark.gpu

BARS = {"bf16x3": 1e-4, "bf16": 2e-2}
DROP_SEED = 20261017


def compact_graph(T, sizes, seed, self_loops=False, repeats=0, type_span=None, extra=0):
    """(adjacency lists, [V, T] in-degrees, V0): components of ``sizes`` nodes (size 1: an isolated node), each a random tree plus a few
    extra edges in both directions.  ``type_span``: a component draws its types from a window of that many consecutive types, so that a
    tile holds only some of them; ``self_loops``: every fifth node sends itself a message; ``repeats``: the first node of each component of
    more than one node receives the same type-0 message from its neighbour ``repeats`` times.  ``extra`` > 0 appends one component of that
    many nodes after the V0 nodes of the rest."""
    rng = np.random.default_rng(seed)
    edges = [[] for _ in range(T)]
    off = 0
    for n in list(sizes) + ([extra] if extra else []):
        span = T if type_span is None else min(type_span, T)
        t0 = int(rng.integers(0, T - span + 1))
        pick = lambda: t0 + int(rng.integers(0, span))
        und = [(off + int(rng.integers(0, i)), off + i) for i in range(1, n)]
        for _ in range(n // 3):
            a, b = rng.choice(n, 2, replace=False)
            und.append((off + int(a), off + int(b)))
        for a, b in und:
            t = pick()
            edges[t] += [(a, b), (b, a)]
        if self_loops:
            for i in range(0, n, 5):
                edges[pick()].append((off + i, off + i))
        if repeats and n > 1:
            edges[0] += [(off + 1, off)] * repeats
        off += n
    adj = [np.asarray(e, np.int32).reshape(-1, 2) for e in edges]
    indeg = np.zeros((off, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg, off - extra


SIZES = (1, 64, 3, 17, 1, 33, 47, 5, 63, 9, 1, 31, 2, 49, 13, 40, 7, 24, 1, 58)


class Case:
    def __init__(self, name, D, T, cell, precision="bf16x3", keep=1.0, **graph):
        self.name, self.D, self.T, self.cell, self.precision, self.keep, self.graph = name, D, T, cell, precision, keep, graph

    @property
    def params(self):
        # tanh on both cells: at a ReLU kink the engine and float64 autograd can take opposite sides (smooth_on_tensor_cores)
        return model(self.cell, self.D, act="tanh", avg=True)


CASES = [Case("nh%d-%s" % (D // 2, cell), D, 4, cell) for D, cell in
         ((16, "GRU"), (32, "RNN"), (48, "GRU"), (64, "RNN"), (80, "GRU"), (96, "RNN"), (112, "GRU"), (128, "RNN"))]
CASES += [
    Case("D100-T4-loops-repeats-GRU", 100, 4, "GRU", self_loops=True, repeats=9),
    Case("D100-T4-loops-repeats-RNN", 100, 4, "RNN", self_loops=True, repeats=9),
    Case("D36-T1-GRU", 36, 1, "GRU", self_loops=True, repeats=5),
    Case("D60-T16-partial-GRU", 60, 16, "GRU", type_span=5, repeats=4),
    # (not DP 128 with 16 types: 128-row tiles there leave the CSR slice in global memory, whose gather adds each message's hi and lo
    # parts in turn, so that layout is not a bit-level reference for it)
    Case("D104-T16-partial-RNN", 104, 16, "RNN", type_span=3, self_loops=True),
    Case("D100-T4-partial-bf16-GRU", 100, 4, "GRU", precision="bf16", type_span=2, repeats=6),
    Case("D64-T4-bf16-RNN", 64, 4, "RNN", precision="bf16", self_loops=True),
]
DROPOUT = [Case("D100-T4-dropout-GRU", 100, 4, "GRU", keep=0.8, self_loops=True, repeats=3),
           Case("D48-T16-dropout-RNN", 48, 16, "RNN", keep=0.7, type_span=4)]


def _weights(p, T, seed=1):
    """The oracle's initialisers with the zero candidate biases drawn, so that every bias enters the forward."""
    rng = np.random.default_rng(seed)
    w = O.init_sparse_weights(p, T, rng)
    for lw in w:
        for k in ("cand_bias", "rnn_bias"):
            if k in lw:
                lw[k] = rng.normal(0, 0.1, lw[k].shape).astype(np.float32)
    return w


def _run(c, adj, indeg, h0, w, g_out, monkeypatch, tiles=None, compact=True):
    """forward states (every layer), the final state and, with ``g_out``, ``d h0`` of one engine run."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM", "GGNN_TC_GATHER_TILES"):
        monkeypatch.delenv(k, raising=False)
    if tiles is not None:
        monkeypatch.setenv("GGNN_TC_GATHER_TILES", str(tiles))
    ren = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}
    dev_w = [{ren.get(k, k): torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).cuda() for k, v in lw.items()} for lw in w]
    eng = PropagationEngine(c.params, c.T, precision=c.precision)
    eng.set_weights(dev_w)
    eng.set_save_for_backward(g_out is not None)
    eng.set_deterministic(True)
    if c.keep < 1.0:
        eng.set_state_dropout(c.keep, DROP_SEED)
    eng.set_graph_sparse(adj, indeg)
    assert eng.plan.startswith("wgmma-%s LOCAL(" % c.precision), eng.plan
    assert ("compact 64-row operand tiles" in eng.plan) == compact, eng.plan
    th0 = torch.from_numpy(h0).cuda()
    out = eng.forward(th0)
    eng.sync_check()
    L = len(c.params["layer_timesteps"])
    res = {"out": out.cpu().numpy(), "layers": [eng.layer_state(l).cpu().numpy() for l in range(L + 1)]}
    if g_out is not None:
        grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in dev_w]
        dh0 = torch.zeros_like(th0)
        eng.backward(torch.from_numpy(g_out).cuda(), grads, dh0)
        eng.sync_check()
        res["dh0"] = dh0.cpu().numpy()
        res["grads"] = [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]
    return res


def _same_bits(got, ref, rows, tag):
    np.testing.assert_array_equal(got["out"][:rows], ref["out"][:rows], err_msg=tag + " out")
    for l, (a, b) in enumerate(zip(got["layers"], ref["layers"])):
        np.testing.assert_array_equal(a[:rows], b[:rows], err_msg="%s layer %d" % (tag, l))
    if "dh0" in got and "dh0" in ref:
        np.testing.assert_array_equal(got["dh0"][:rows], ref["dh0"][:rows], err_msg=tag + " d h0")


@pytest.mark.parametrize("case", [c.name for c in CASES])
def test_compact_timestep_matches_the_128_row_layout(case, monkeypatch):
    c = next(x for x in CASES if x.name == case)
    adj, indeg, V = compact_graph(c.T, SIZES, seed=c.D + c.T, **c.graph)
    adj_x, indeg_x, V_x = compact_graph(c.T, SIZES, seed=c.D + c.T, extra=100, **c.graph)
    assert V_x == V and all(np.array_equal(a, b[:len(a)]) for a, b in zip(adj, adj_x))
    rng = np.random.default_rng(c.D)
    h0_x = rng.normal(0, 1, (indeg_x.shape[0], c.D)).astype(np.float32)
    h0 = np.ascontiguousarray(h0_x[:V])
    w = _weights(c.params, c.T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    g_out_x = np.zeros_like(h0_x)
    g_out_x[:V] = g_out

    new = _run(c, adj, indeg, h0, w, g_out, monkeypatch)
    old = _run(c, adj_x, indeg_x, h0_x, w, g_out_x, monkeypatch, compact=False)
    _same_bits(new, old, V, "%s compact vs 128-row" % case)
    for tiles in (2, 3):
        _same_bits(_run(c, adj, indeg, h0, w, g_out, monkeypatch, tiles=tiles), new, V, "%s %d gather tiles" % (case, tiles))

    ref_out, ref_dh0, ref_gw = _autograd_reference(c.params, c.T, w, adj, indeg, h0, g_out)
    scale = float(np.max(np.abs(ref_out)))
    err = float(np.max(np.abs(new["out"] - ref_out))) / scale
    assert err < BARS[c.precision], (case, err)
    if c.precision == "bf16x3":
        _cmp(new["dh0"], ref_dh0, case + " d h0")
        for l, (gw, rw) in enumerate(zip(new["grads"], ref_gw)):
            for k in rw:
                _cmp(gw["cand_kernel" if k == "rnn_kernel" else "cand_bias" if k == "rnn_bias" else k], rw[k], "%s layer %d %s" % (case, l, k))


@pytest.mark.parametrize("case", [c.name for c in DROPOUT])
def test_compact_timestep_with_state_dropout(case, monkeypatch):
    import torch
    c = next(x for x in DROPOUT if x.name == case)
    adj, indeg, V = compact_graph(c.T, SIZES, seed=c.D + c.T, **c.graph)
    h0 = np.random.default_rng(c.D).normal(0, 1, (V, c.D)).astype(np.float32)
    w = _weights(c.params, c.T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    new = _run(c, adj, indeg, h0, w, g_out, monkeypatch)
    for tiles in (2, 3):
        got = _run(c, adj, indeg, h0, w, g_out, monkeypatch, tiles=tiles)
        _same_bits(got, new, V, "%s %d gather tiles" % (case, tiles))
        for l, (ga, gb) in enumerate(zip(got["grads"], new["grads"])):
            for k in ga:
                np.testing.assert_array_equal(ga[k], gb[k], err_msg="%s %d gather tiles layer %d d %s" % (case, tiles, l, k))
    refs = O.sparse_propagation_torch(h0, adj, indeg, w, c.params, dtype=torch.float64, return_all_layers=True,
                                      state_dropout=(c.keep, DROP_SEED))
    for l, (a, r) in enumerate(zip(new["layers"], refs)):
        r = r.numpy()
        err = float(np.max(np.abs(a - r))) / float(np.max(np.abs(r)))
        assert err < BARS[c.precision], (case, l, err)
