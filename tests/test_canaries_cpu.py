"""CPU: the memory canaries of tests/test_gpu_canaries.py -- their helpers, their cases and the plans those cases reach, without a GPU.

The GPU file poisons whole connected components with a payload NaN and checks that the clean ones keep their bits, puts every caller
buffer between NaN guard bands, runs one engine through a NaN batch and NaN weights, and checks the aliasing rule of ``ggnn_forward``.
Those checks only mean something if the batches have the shapes they claim: here every new batch is built through the host-only prepare
calls at 132 SMs (an H100 SXM) and must reach its plan, every isolation case must have clean and poisoned components in the places the
GPU file relies on (a clean component in a tile shared with poisoned ones, one in the last tile, poisoned ones on both sides of a tile cut
on GLOBAL and streaming plans), ``guarded`` must detect a one-word overwrite at either end, and the header must state the aliasing rule.
"""
import os
import re

import numpy as np
import pytest

from tests import gcn_oracle as G
from tests.test_backward_plans_cpu import (DENSE_CASES, DENSE_T, EDGE_SHAPES, FORCE_GLOBAL, GCN_CASES, GCN_LAYERS, PLAN_MATRIX,
                                           TC_STREAM, Case, component_graph, dense_batch, dense_params, gcn_batch, model, plan_matches,
                                           sparse_batch)

NUM_SMS = 132
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ---------------------------------------------------------------------------------------------------------------- guard bands
PAYLOAD = 0x7FC0DEAD          # a quiet NaN with a payload: arithmetic on the GPU produces 0x7fffffff, only moves / neg / abs keep this one
BAND = 128 * 512              # floats on each side: a 128-row tile at hidden 512 over-running stays inside the band; a multiple of 64


class Guarded:
    """One flat buffer filled with ``PAYLOAD`` (through an int32 view), ``BAND`` floats of it on each side of a contiguous fp32 view of
    ``n`` elements.  ``view`` is what a call gets; ``bands_intact()`` compares both bands with the payload bit for bit."""

    def __init__(self, n, device="cuda"):
        import torch
        self.n = int(n)
        self.raw = torch.full((self.n + 2 * BAND,), PAYLOAD, dtype=torch.int32, device=device)
        self.view = self.raw.view(torch.float32)[BAND:BAND + self.n]

    def bands_intact(self):
        import torch
        lo, hi = self.raw[:BAND], self.raw[BAND + self.n:]
        return bool(torch.all(lo == self.raw[0]).item()) and bool(torch.all(hi == self.raw[0]).item()) and int(self.raw[0].item()) & 0xFFFFFFFF == PAYLOAD


def guarded(n, device="cuda"):
    return Guarded(n, device)


def has_payload(t):
    """True when a word of ``t`` holds the payload under either sign: guard or prefill bytes were copied or stored there."""
    import torch
    bits = t.detach().contiguous().view(torch.int32) & 0x7FFFFFFF
    return bool(torch.any(bits == PAYLOAD).item())


def payload_nan(shape):
    """A float32 NumPy array of the payload NaN."""
    return np.full(shape, PAYLOAD, np.uint32).view(np.float32)


# ---------------------------------------------------------------------------------------------------------------- components
def components(V, edges):
    """Weakly connected components (labels [V], count) of ``edges``: an ``[E, 2]`` array or a list of them (one per edge type)."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    e = np.concatenate([np.asarray(a, np.int64).reshape(-1, 2) for a in (edges if isinstance(edges, (list, tuple)) else [edges])], axis=0)
    m = sp.coo_matrix((np.ones(e.shape[0]), (e[:, 0], e[:, 1])), shape=(V, V))
    n, lab = connected_components(m, directed=True, connection="weak")
    return lab, n


def poisoned_components(n, labels=None, tile_start=None):
    """The first, the last and every third component from the second on, the one before the last excepted (so that a last tile of
    several components holds a clean one): clean and poisoned components alternate through every tile.  With ``labels`` and the plan's
    ``tile_start`` also the component holding the last row before the first tile cut and the one holding the first row after the second
    (GLOBAL and streaming plans cut through the batch by rows)."""
    bad = {0, n - 1} | set(range(1, n - 2, 3))
    if labels is not None and tile_start is not None and len(tile_start) > 2:
        cuts = [int(c) for c in tile_start[1:-1]]
        bad |= {int(labels[cuts[0] - 1]), int(labels[cuts[min(1, len(cuts) - 1)]])}
    return np.array(sorted(bad), np.int64)


def layout(labels, poisoned, tile_start):
    """What an isolation case looks like in its plan: counts; whether a clean component shares a tile with a poisoned one; whether the
    last tile holds a clean component, or only one component (the last, which is poisoned); whether some tile cut has a poisoned row right
    before it and a clean row in the tile after it, and some cut a poisoned row right after it and a clean row in the tile before it."""
    bad = np.isin(labels, poisoned)
    tiles = [(int(a), int(b)) for a, b in zip(tile_start[:-1], tile_start[1:]) if b > a]
    mixed = any(bad[a:b].any() and (~bad[a:b]).any() for a, b in tiles)
    last_clean = bool((~bad[tiles[-1][0]:tiles[-1][1]]).any()) if tiles else False
    last_single = len(set(labels[tiles[-1][0]:tiles[-1][1]].tolist())) == 1 if tiles else True
    pairs = list(zip(tiles[:-1], tiles[1:]))
    return {"clean": int(len(set(labels[~bad].tolist()))), "poisoned": int(len(set(labels[bad].tolist()))), "mixed_tile": mixed,
            "last_tile_clean": last_clean, "last_tile_single": last_single,
            "tile_before_last_clean": len(tiles) > 1 and bool((~bad[tiles[-2][0]:tiles[-2][1]]).any()),
            "cut_poisoned_then_clean": any(bad[t[0] - 1] and (~bad[t[0]:t[1]]).any() for _, t in pairs),
            "cut_clean_then_poisoned": any(bad[t[0]] and (~bad[s[0]:s[1]]).any() for s, t in pairs), "tiles": len(tiles),
            "single_component_tiles": all(len(set(labels[a:b].tolist())) == 1 for a, b in tiles)}


# ---------------------------------------------------------------------------------------------------------------- the cases
WIDE_STEP = r"^fp32-stepwise "
ATT_LOCAL = r"^fp32-ffma\+attention LOCAL\("


def _isolation_sparse():
    """(case, state keep probability): every PLAN_MATRIX family, the edge shapes at T = 1 / 17 / 32 and the zero-step layer, attention on
    GLOBAL and fp32 LOCAL, CudnnCompatibleGRUCell (in PLAN_MATRIX), hidden 260 and 512 (per-timestep fp32 and streaming), dropout 0.8."""
    out = [(c, 1.0) for c in PLAN_MATRIX]
    out += [(c, 1.0) for c in EDGE_SHAPES if re.match(r"^(T1|T17|T32)-|^zero-step-", c.name)]
    out.append((Case("ffma-local-attention-D36", model("GRU", 36, act="tanh", attention=True), 4, "mol24", "fp32", {}, ATT_LOCAL), 1.0))
    for D in (260, 512):
        out.append((Case("wide-step-gru-D%d" % D, model("GRU", D, act="tanh"), 4, "mol24", "fp32", {}, WIDE_STEP), 1.0))
        out.append((Case("wide-stream-rnn-D%d" % D, model("RNN", D, act="tanh"), 4, "mol24", "bf16x3", {}, TC_STREAM), 1.0))
    out.append((Case("drop-ffma0-gru-D36", model("GRU", 36), 4, "mol24", "fp32", {"GGNN_FFMA_VARIANT": "0"}, r"^fp32-ffma LOCAL\("), 0.8))
    out.append((Case("drop-tc-global-gru-D100", model("GRU", 100, act="tanh"), 4, "mol24", "bf16x3", FORCE_GLOBAL, r"^wgmma-bf16x3 GLOBAL\("), 0.8))
    return out


ISOLATION_SPARSE = _isolation_sparse()


def end_of_batch_covered(lay):
    """A clean component in the last tile -- or, where the plan gives the (poisoned) last component a tile of its own, so that no clean one
    can share it, a clean component in the tile before.  Small batches get one component per tile (the planner spreads them over the
    SMs); test_some_last_tiles_hold_clean_and_poisoned_components requires the shared case on the batches where the last tile is shared."""
    return lay["last_tile_clean"] or (lay["last_tile_single"] and lay["tile_before_last_clean"])
ISOLATION_SPARSE_BY_NAME = {c.name: (c, k) for c, k in ISOLATION_SPARSE}
GLOBAL_OR_STREAM = re.compile(r" (GLOBAL|STREAM)\(|^fp32-stepwise ")


def sparse_isolation_batch(c, tile_start):
    """(adj, indeg, h0, labels, poisoned component ids) of a sparse case whose plan has ``tile_start``."""
    adj, indeg, h0 = sparse_batch(c.batch, c.params["hidden_size"], c.T)
    labels, n = components(indeg.shape[0], adj)
    return adj, indeg, h0, labels, poisoned_components(n, labels, tile_start)


def dense_isolation_batch(D, weighted):
    """(A [b, T, v, v], h0 [b, v, D], graph ids poisoned): whole graphs are the unit here, as the dense model's batched matmul mixes no two."""
    A, h0 = dense_batch(D, weighted)
    return A, h0, poisoned_components(A.shape[0])


SMALL_GCN_COMPONENTS = 10


def gcn_isolation_batch(D, kind, tile_start=None, seed=0):
    """``gcn_batch`` with, for the GLOBAL case's 300-node random graph, ten molecule-sized components appended.  Returns (V, lst, w, ks,
    bs, h0, labels, poisoned runs): the components case poisons its usual set; the GLOBAL case once the big component (and its isolated
    nodes' neighbours stay clean), once the small ones."""
    V, lst, w, ks, bs, h0 = gcn_batch(D, kind, seed)
    if kind == "random":
        rng = np.random.default_rng(1000 + D)
        Vs, ls, ws = G.component_list(list(rng.integers(8, 30, SMALL_GCN_COMPONENTS)), rng)
        lst = np.concatenate([lst, ls + V], axis=0)
        w = np.concatenate([w, ws]).astype(np.float32)
        h0 = np.concatenate([h0, rng.normal(0, 1, (Vs, D)).astype(np.float32)], axis=0)
        V += Vs
    labels, n = components(V, lst)
    if kind == "random":
        big = int(np.bincount(labels).argmax())
        small = np.array(sorted(set(labels[V - (V - 300):].tolist())), np.int64)
        runs = [np.array([big], np.int64), small]
    else:
        runs = [poisoned_components(n, labels, tile_start)]
    return V, lst, w, ks, bs, h0, labels, runs


# the batches of the leftovers sequence (section C of the GPU file): A, then a larger P, then a smaller B
LEFTOVER_FAMILIES = ["ffma0-local-gru-D100", "ffma-global-gru-D100", "tc-local64-gru-D100", "tc-global-rnn-D100", "stream-gru-D132",
                     "ffma-local-cudnn-D100", "ffma-global-attention-D36"]
LEFTOVER_BATCHES = {"A": "mol24", "P": "mol160", "B": "mol10"}

# guard-band shapes (section B): (name, V target, hidden, precision, env, plan)
GUARD_SHAPES = [("V1-D4", 1, 4, "fp32", {}, r"^fp32-ffma LOCAL\("), ("V15-D20", 15, 20, "bf16x3", {}, r"^wgmma-bf16x3 LOCAL\("),
                ("V17-D36", 17, 36, "fp32", FORCE_GLOBAL, r"^fp32-ffma GLOBAL\("), ("V63-D100", 63, 100, "bf16x3", FORCE_GLOBAL, r"^wgmma-bf16x3 GLOBAL\("),
                ("V65-D132", 65, 132, "bf16x3", {}, TC_STREAM), ("V129-D252", 129, 252, "fp32", {}, r"^fp32-ffma LOCAL\("),
                ("V129-D260", 129, 260, "fp32", {}, WIDE_STEP), ("V10000-D512", 10000, 512, "bf16x3", {}, TC_STREAM),
                ("V0-D36", 0, 36, "fp32", {}, r"")]


def chain_batch(V, T=4, seed=0):
    """Components of 1 to 7 nodes (chains with both directions, types uniform over ``T``) totalling exactly V nodes: the last tile of
    every plan ends at an awkward row."""
    rng = np.random.default_rng(seed + V)
    sizes, left = [], V
    while left > 0:
        n = int(min(left, rng.integers(1, 8)))
        sizes.append(n)
        left -= n
    edges, off = [], 0
    for n in sizes:
        edges += [(off + i, off + i + 1) for i in range(n - 1)]
        off += n
    e = np.asarray(edges, np.int64).reshape(-1, 2)
    types = rng.integers(0, T, e.shape[0])
    adj = [np.concatenate([e[types == t], e[types == t][:, ::-1]], axis=0).astype(np.int32).reshape(-1, 2) for t in range(T)]
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg


def guard_params(D):
    return model("GRU", D, act="tanh")


# ---------------------------------------------------------------------------------------------------------------- tests
def _host_plan(c, adj, indeg):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    g = PreparedGraph.host_only(c.params, c.T, adj, indeg, precision=c.precision, num_sms=NUM_SMS, save_for_backward=True)
    return g.info()["plan"], g.arrays(c.T)["tile_start"]


@pytest.mark.parametrize("name", sorted(ISOLATION_SPARSE_BY_NAME))
def test_sparse_isolation_case_reaches_its_plan_and_has_both_kinds_of_component(name, monkeypatch):
    c, _ = ISOLATION_SPARSE_BY_NAME[name]
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    adj, indeg, _ = sparse_batch(c.batch, c.params["hidden_size"], c.T)
    plan, ts = _host_plan(c, adj, indeg)
    _, _, _, labels, bad = sparse_isolation_batch(c, ts)
    assert plan_matches(plan, c.plan), (c.plan, plan)
    lay = layout(labels, bad, ts)
    assert lay["clean"] >= 2 and lay["poisoned"] >= 2, lay
    assert lay["mixed_tile"], lay
    assert end_of_batch_covered(lay), lay
    if GLOBAL_OR_STREAM.search(plan):
        assert lay["cut_poisoned_then_clean"] and lay["cut_clean_then_poisoned"], lay


@pytest.mark.parametrize("name,precision,D,weighted,pattern", [c for c in DENSE_CASES if not c[3]], ids=lambda x: str(x))
def test_dense_isolation_case_has_both_kinds_of_graph(name, precision, D, weighted, pattern):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    A, _, bad = dense_isolation_batch(D, weighted)
    g = PreparedGraph.host_only_dense(dense_params(D), DENSE_T, A, precision=precision, num_sms=NUM_SMS, save_for_backward=True)
    assert plan_matches(g.info()["plan"], pattern)
    b, v = A.shape[0], A.shape[2]
    graph_of_row = np.repeat(np.arange(b), v)
    lay = layout(graph_of_row, bad, g.arrays(DENSE_T)["tile_start"])
    assert lay["clean"] >= 2 and lay["poisoned"] >= 2 and end_of_batch_covered(lay), lay
    assert lay["mixed_tile"] or lay["single_component_tiles"], lay   # a tile of one graph cannot mix: the unit is the graph


@pytest.mark.parametrize("name,precision,D,kind,keep,env,pattern", GCN_CASES, ids=[c[0] for c in GCN_CASES])
def test_gcn_isolation_case_reaches_its_plan(name, precision, D, kind, keep, env, pattern, monkeypatch):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    V, lst, w = gcn_isolation_batch(D, kind)[:3]
    g = PreparedGraph.host_only_gcn(D, GCN_LAYERS, V, lst, w, use_bias=True, precision=precision, num_sms=NUM_SMS, save_for_backward=True)
    plan = g.info()["plan"]
    assert plan_matches(plan, pattern), (pattern, plan)
    ts = g.arrays(1)["tile_start"]
    labels, runs = gcn_isolation_batch(D, kind, ts)[6:]
    for bad in runs:
        lay = layout(labels, bad, ts)
        assert lay["clean"] >= 1 and lay["poisoned"] >= 1, lay
        if kind == "components":
            assert lay["clean"] >= 2 and lay["poisoned"] >= 2 and lay["mixed_tile"] and end_of_batch_covered(lay), lay
    if kind == "random":
        assert len(set(labels[300:].tolist())) == SMALL_GCN_COMPONENTS
        lay = layout(labels, runs[0], ts)
        assert lay["cut_poisoned_then_clean"] and lay["clean"] >= SMALL_GCN_COMPONENTS, lay


@pytest.mark.parametrize("name", LEFTOVER_FAMILIES)
def test_leftover_batches_grow_then_shrink_on_one_plan(name, monkeypatch):
    from tests.test_backward_plans_cpu import SPARSE_CASES
    c = SPARSE_CASES[name]
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    sizes = {}
    for tag, kind in LEFTOVER_BATCHES.items():
        adj, indeg, _ = sparse_batch(kind, c.params["hidden_size"], c.T)
        plan, _ = _host_plan(c, adj, indeg)
        assert plan_matches(plan, c.plan), (tag, c.plan, plan)
        sizes[tag] = (indeg.shape[0], sum(a.shape[0] for a in adj))
    assert sizes["P"][0] > sizes["A"][0] > sizes["B"][0] and sizes["P"][1] > sizes["A"][1] > sizes["B"][1], sizes


@pytest.mark.parametrize("shape", GUARD_SHAPES, ids=[s[0] for s in GUARD_SHAPES])
def test_guard_band_shapes_reach_their_plans(shape, monkeypatch):
    name, V, D, precision, env, pattern = shape
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    adj, indeg = chain_batch(V)
    assert indeg.shape[0] == V
    c = Case(name, guard_params(D), 4, None, precision, env, pattern)
    plan, ts = _host_plan(c, adj, indeg)
    assert plan_matches(plan, pattern), (pattern, plan)
    assert ts[-1] == V


def test_gcn_aliasing_batch_reaches_the_fp32_and_local_plans():
    """The GCN forward-refusal and backward-alias tests of the GPU file run one-layer batches at the reference's h12_l1 shape (hidden 12)
    on the LOCAL wgmma kernel and on the fp32 kernel."""
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    V, lst, w, _, _, _ = gcn_batch(12, "components")
    for prec, pat in (("bf16x3", r"^gcn-wgmma-bf16x3 LOCAL\("), ("fp32", r"^gcn-fp32-ffma GLOBAL\(")):
        g = PreparedGraph.host_only_gcn(12, 1, V, lst, w, precision=prec, num_sms=NUM_SMS, save_for_backward=True)
        assert plan_matches(g.info()["plan"], pat), g.info()["plan"]


def test_guarded_self_test_on_cpu_tensors():
    import torch
    n = 1001
    g = guarded(n, device="cpu")
    assert g.view.dtype == torch.float32 and g.view.is_contiguous() and g.view.numel() == n
    assert g.view.data_ptr() % 16 == 0 and (g.view.data_ptr() - g.raw.data_ptr()) == BAND * 4 and BAND % 64 == 0 and BAND >= 128 * 512
    assert bool(torch.all(torch.isnan(g.view))) and has_payload(g.view) and has_payload(-g.view) and has_payload(g.view.abs())
    assert int(g.raw[0].item()) & 0xFFFFFFFF == PAYLOAD and g.bands_intact()
    assert not has_payload(torch.full((4,), float("nan")))          # an arithmetic NaN is not the payload
    g.view.zero_()
    assert g.bands_intact() and not has_payload(g.view)
    raw = g.raw.view(torch.float32)
    for idx in (BAND - 1, BAND + n):                                   # one word before the view, one after
        keep = g.raw[idx].clone()
        raw[idx] = 0.0
        assert not g.bands_intact(), idx
        g.raw[idx] = keep
        assert g.bands_intact()
    np.testing.assert_array_equal(payload_nan(3).view(np.uint32), np.full(3, PAYLOAD, np.uint32))


def test_header_states_the_aliasing_rule():
    with open(os.path.join(ROOT, "include", "ggnn_b200.h")) as f:
        h = re.sub(r"\s+", " ", f.read())
    assert "must not overlap those at h0" in h and "GGNN_EINVAL naming both pointers" in h
    assert "both must stay unchanged until the backward has run" in h
    assert "d_h0 may be d_h_out or overlap it" in h


def test_components_of_the_edge_shape_graphs():
    adj, indeg = component_graph(4, seed=4)
    lab, n = components(indeg.shape[0], adj)
    assert lab[0] != lab[1] and lab[2] == lab[3] and lab[1] != lab[2] and n > 10
    bad = poisoned_components(n)
    assert bad[0] == 0 and bad[-1] == n - 1 and len(bad) >= 3


def test_some_last_tiles_hold_clean_and_poisoned_components(monkeypatch):
    """Where the batch's last tile holds several components, the poisoned last component shares it with a clean one: the 1024-molecule
    LOCAL case, the GLOBAL wgmma case and the streaming cases (128-row tiles cut by rows)."""
    shared = []
    for name in ("tc-local128-gru-D100", "tc-global-gru-D100", "stream-gru-D132", "wide-stream-rnn-D512"):
        c, _ = ISOLATION_SPARSE_BY_NAME[name]
        for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM", "GGNN_FFMA_VARIANT"):
            monkeypatch.delenv(k, raising=False)
        for k, v in c.env.items():
            monkeypatch.setenv(k, v)
        adj, indeg, _ = sparse_batch(c.batch, c.params["hidden_size"], c.T)
        _, ts = _host_plan(c, adj, indeg)
        labels, bad = sparse_isolation_batch(c, ts)[3:]
        lay = layout(labels, bad, ts)
        assert not lay["last_tile_single"] and lay["last_tile_clean"], (name, lay)
        shared.append(name)
    assert len(shared) == 4
