"""CPU: the batches, score regimes and plans of tests/test_gpu_attention_edges.py, and the float64 oracle on them.

Propagation attention (sparse:170-196) runs four pieces of CUDA of its own: the softmax pre-pass of the fp32 forward (one warp per target:
scores, max, exp, sum, normalise), the probability-weighted gather, ``attention_bwd_target_kernel`` (softmax backward, ``d a_t`` through a
16-slot shared array, ``d h[target]`` in an 8-slot-per-lane column loop) and ``attention_bwd_source_kernel`` (``d h[source]`` through the
source-keyed CSR).  Molecules reach none of their edges: an in-degree of about 4, at most 4 edge types, no self-loops, scores of a few
units.  The batches here do:

* ``hubs``: targets with exactly 1, 31, 32, 33, 64, 65 and 300 incoming messages over at least three types (duplicate edges, so that
  every component stays within a 32-row fp32 tile), isolated nodes;
* ``big_hub``: one component of more than 1000 nodes around a target of in-degree >= 1000, larger than any fp32 tile (GLOBAL by itself);
* ``self_dup``: a node whose only message is a self-loop, self-loops beside other messages, one (source, target) pair twice in a type,
  one pair under two types;
* ``t16_all`` / ``t16_ends`` / ``t1``: 16 edge types (the most attention takes) all present, 16 types of which only 0 and 15 occur, and a
  single type.

Score regimes (``h0`` scale and ``edge_type_attention_weights``): ``mild`` (scores of a few units), ``large`` (step-0 scores >= 90: fp32
``exp`` without the max-shift overflows), ``negative`` (a node with >= 2 messages whose step-0 scores are all <= -90: without the shift
its weights underflow to 0), ``a_zero`` (one type's weight 0) and ``a_negative`` (two types' weights < 0).

Tests: the batches have the shapes and score extremes they claim; the oracle statements (float64 loops, NumPy, torch and the plain-C
restatement) agree to 1e-12 on them; every GPU case reaches its plan through the host-only prepare calls at 132 SMs (an H100 SXM);
17 edge types with attention are refused.
"""
import functools
import os
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from oracle import ggnn_oracle as O
from tests.test_backward_plans_cpu import component_graph, model

NUM_SMS = 132
HUB_DEGREES = (1, 31, 32, 33, 64, 65, 300)
BIG_HUB_DEGREE = 1100
BOUND = 90.0          # |step-0 score| the large / negative regimes reach: exp(90) > FLT_MAX, exp(-90) < 1e-39


# ---------------------------------------------------------------------------------------------------------------- batch kinds
def wire(V, T, edges):
    """(src, tgt, type) triples -> the reference wire format: per-type ``[E_t, 2]`` int32 lists (in triple order) and the ``[V, T]``
    in-degree table."""
    e = np.asarray(edges, np.int64).reshape(-1, 3)
    adj = [np.ascontiguousarray(e[e[:, 2] == t][:, :2], dtype=np.int32) for t in range(T)]
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg


def _filler(rng, off, count, T, edges, max_size=20):
    """Random small trees with a few extra edges (both directions, uniform types) from node ``off`` on; returns the next free node."""
    end = off + count
    while off < end:
        n = min(int(rng.integers(3, max_size)), end - off)
        if n < 2:
            return off + n
        und = [(off + int(rng.integers(0, i)), off + i) for i in range(1, n)]
        for _ in range(n // 4):
            a, b = rng.choice(n, 2, replace=False)
            und.append((off + int(a), off + int(b)))
        for a, b in und:
            t = int(rng.integers(0, T))
            edges += [(a, b, t), (b, a, t)]
        off += n
    return off


def hubs(seed, T=4):
    """Nodes 0, 1 isolated; then per degree k of HUB_DEGREES a component whose hub (its first node) receives exactly k messages from at
    most 20 sources (duplicates), types cycling over min(T, 3 or 4); each source also receives one message from the hub; then fillers.
    Every component has at most 21 nodes."""
    rng = np.random.default_rng(seed)
    edges, off = [], 2
    for k in HUB_DEGREES:
        ns = min(k, 12 if k < 300 else 20)
        hub, srcs = off, list(range(off + 1, off + 1 + ns))
        order = rng.permutation(k)
        for j in order:
            edges.append((srcs[j % ns], hub, int(j % min(T, 3 if k < 300 else 4))))
        for s in srcs:
            edges.append((hub, s, int(rng.integers(0, T))))
        off += 1 + ns
    off = _filler(rng, off, 200, T, edges)
    return wire(off, T, edges)


def big_hub(seed, T=4):
    """One component: node 0 receives BIG_HUB_DEGREE messages, one from each of nodes 1 .. BIG_HUB_DEGREE, types cycling; a chain among
    the sources; then fillers."""
    rng = np.random.default_rng(seed)
    edges = [(s, 0, s % T) for s in range(1, BIG_HUB_DEGREE + 1)]
    edges += [(s, s + 1, int(rng.integers(0, T))) for s in range(1, BIG_HUB_DEGREE)]
    edges += [(0, s, int(rng.integers(0, T))) for s in range(1, BIG_HUB_DEGREE + 1, 7)]
    off = _filler(rng, BIG_HUB_DEGREE + 1, 200, T, edges)
    return wire(off, T, edges)


SELF_ONLY, SELF_PLUS, DUP_TGT, TWO_TYPES_TGT = 2, 5, 9, 13   # node ids the self_dup shape test looks at


def self_dup(seed, T=4):
    """Nodes 0, 1 isolated.  Node 2: only a self-loop.  Nodes 3-6: a component where 5 has a self-loop and two other messages and 6 a
    self-loop of two types.  Nodes 7-10: (8 -> 9) twice in type 1.  Nodes 11-14: (12 -> 13) in types 0 and 2.  Then fillers with a
    self-loop on every fifth node."""
    rng = np.random.default_rng(seed)
    edges = [(2, 2, 0),
             (3, 4, 0), (4, 3, 0), (5, 5, 1), (3, 5, 0), (4, 5, 2), (5, 3, 1), (6, 6, 0), (6, 6, 3 % T), (5, 6, 2 % T),
             (7, 8, 0), (8, 9, 1), (8, 9, 1), (10, 9, 0), (9, 10, 3 % T), (8, 7, 2 % T),
             (11, 12, 0), (12, 13, 0), (12, 13, 2 % T), (13, 14, 1), (14, 13, 1), (13, 11, 0)]
    fill = []
    off = _filler(rng, 15, 200, T, fill)
    edges += fill + [(v, v, int(rng.integers(0, T))) for v in range(15, off, 5)]
    return wire(off, T, edges)


def t16_all(seed):
    """component_graph at 16 types (every type occurs), plus a target receiving one message of each of the 16 types."""
    adj, indeg = component_graph(16, V_target=300, seed=seed)
    V = indeg.shape[0]
    edges = [(int(s), int(d), t) for t, a in enumerate(adj) for s, d in a]
    edges += [(V + 1 + (t % 8), V, t) for t in range(16)] + [(V, V + 1 + j, j) for j in range(8)]
    return wire(V + 9, 16, edges)


def t16_ends(seed):
    """16 types, only types 0 and 15 occur."""
    rng = np.random.default_rng(seed)
    edges = []
    off = _filler(rng, 2, 300, 2, edges)
    return wire(off, 16, [(s, d, 15 * t) for s, d, t in edges])


def t1(seed):
    adj, indeg = component_graph(1, V_target=300, seed=seed)
    return adj, indeg


KINDS = {"hubs": (hubs, 4), "big_hub": (big_hub, 4), "self_dup": (self_dup, 4), "t16_all": (t16_all, 16), "t16_ends": (t16_ends, 16),
         "t1": (t1, 1)}


@functools.lru_cache(maxsize=None)
def batch(kind, seed=0):
    """(adjacency lists, in-degree table, T) of a batch kind."""
    fn, T = KINDS[kind]
    adj, indeg = fn(seed) if T in (1, 16) else fn(seed, T)
    return adj, indeg, T


# ---------------------------------------------------------------------------------------------------------------- score regimes
REGIMES = ("mild", "large", "negative", "a_zero", "a_negative")


def regime_h0(regime, V, D, seed=0):
    """``mild`` (and the a_t regimes): N(0, sigma) with sqrt(D) sigma^2 = 2, step-0 scores of a few units.  ``large`` / ``negative``: a
    common offset c (D c^2 = 120) plus N(0, 0.5) noise: every <h[src], h[tgt]> is about 120 +- 10."""
    rng = np.random.default_rng(1000 + seed + D)
    if regime in ("large", "negative"):
        return (np.sqrt(120.0 / D) + rng.normal(0, 0.5, (V, D))).astype(np.float32)
    return rng.normal(0, np.sqrt(2.0 / np.sqrt(D)), (V, D)).astype(np.float32)


def regime_weights(p, T, regime, seed=1):
    """The oracle's initialisers with the zero candidate biases drawn (every bias enters the forward) and the attention weights of the
    regime: mild U(0.5, 1.5); large 1 + U(0, 0.2); negative -(1 + U(0, 0.2)); a_zero type 1 -> 0; a_negative types 0 and 2 -> < 0."""
    rng = np.random.default_rng(seed)
    w = O.init_sparse_weights(p, T, rng, attention_scale=0.5)
    for lw in w:
        for k in ("cand_bias", "rnn_bias"):
            if k in lw:
                lw[k] = rng.normal(0, 0.1, lw[k].shape).astype(np.float32)
        a = lw["edge_type_attention_weights"]
        if regime in ("large", "negative"):
            a[:] = (1.0 + 0.2 * rng.uniform(0, 1, T)) * (1 if regime == "large" else -1)
        elif regime == "a_zero":
            a[1 % T] = 0.0
        elif regime == "a_negative":
            a[0] = -0.8
            a[2 % T] = -1.3
    return w


def step0_scores(h0, adj, a):
    """float64 step-0 scores of every message, and its target."""
    h = np.asarray(h0, np.float64)
    src, tgt, typ = O.message_arrays(adj)
    return np.einsum("md,md->m", h[src], h[tgt]) * np.asarray(a, np.float64)[typ], tgt


# ---------------------------------------------------------------------------------------------------------------- the GPU cases
def att_model(D, cell="GRU", act="tanh", layer_timesteps=(2, 1), residual_connections=None, bias=True, avg=True):
    return model(cell, D, layer_timesteps=layer_timesteps, residual_connections=residual_connections, act=act, bias=bias, avg=avg,
                 attention=True)


ATT_LOCAL_64 = r"^fp32-ffma\+attention LOCAL\(.* rows/tile<=64 warps=8 colsplit=1 "    # variant 0
ATT_LOCAL_32 = r"^fp32-ffma\+attention LOCAL\(.* rows/tile<=32 warps=8 colsplit=2 "    # variant 1
ATT_LOCAL = r"^fp32-ffma\+attention LOCAL\("
ATT_GLOBAL = r"^fp32-ffma\+attention GLOBAL\("
ATT_CUDNN_LOCAL = r"^fp32-ffma\+attention\+cudnn-gru LOCAL\("
ATT_CUDNN_GLOBAL = r"^fp32-ffma\+attention\+cudnn-gru GLOBAL\("
FORCE_GLOBAL = {"GGNN_FORCE_GLOBAL": "1"}
VARIANT0 = {"GGNN_FFMA_VARIANT": "0"}


class Case:
    def __init__(self, name, params, kind, regime, env, plan, group, state_keep=1.0):
        self.name, self.params, self.kind, self.regime, self.env, self.plan = name, params, kind, regime, env, plan
        self.group, self.state_keep = group, state_keep

    @property
    def D(self):
        return self.params["hidden_size"]

    def __repr__(self):
        return self.name


SWEEP_EXTRA = (4, 12, 36, 132, 252, 256)
SWEEP_VARIANT0 = (4, 12, 36, 128)


def _cases():
    out = []
    # hidden sweep: every accepted hidden size on the default plan (variant 1 LOCAL: the hubs batch is small and its components fit 32
    # rows), at six of them GLOBAL, and the 64-row variant 0 where it exists (hidden <= 128: its shared memory does not fit above)
    for D in range(4, 257, 4):
        out.append(Case("sweep-D%d" % D, att_model(D), "hubs", "mild", {}, ATT_LOCAL_32, "hidden sweep"))
    for D in SWEEP_EXTRA:
        out.append(Case("sweep-global-D%d" % D, att_model(D), "hubs", "mild", FORCE_GLOBAL, ATT_GLOBAL, "hidden sweep"))
    for D in SWEEP_VARIANT0:
        out.append(Case("sweep-v0-D%d" % D, att_model(D), "hubs", "mild", VARIANT0, ATT_LOCAL_64, "hidden sweep"))
    # degree and topology
    for kind in KINDS:
        for D in (36, 132):
            if kind != "big_hub":
                out.append(Case("%s-local-D%d" % (kind, D), att_model(D), kind, "mild", {}, ATT_LOCAL, "degree and topology"))
            out.append(Case("%s-global-D%d" % (kind, D), att_model(D), kind, "mild", FORCE_GLOBAL if kind != "big_hub" else {}, ATT_GLOBAL,
                            "degree and topology"))
    # score regimes
    for regime in REGIMES[1:]:
        for D in (36, 256):
            out.append(Case("%s-D%d" % (regime, D), att_model(D), "hubs", regime, {}, ATT_LOCAL,
                            "large / negative scores" if regime in ("large", "negative") else "a_t = 0 / a_t < 0"))
    # feature crosses
    crosses = {"dropout": (lambda D: att_model(D), 0.8),
               "cudnn": (lambda D: att_model(D, cell="CudnnCompatibleGRUCell"), 1.0),
               "rnn-tanh": (lambda D: att_model(D, cell="RNN"), 1.0),
               "zero-step": (lambda D: att_model(D, layer_timesteps=(2, 0, 1), residual_connections={"2": [1, 2]}), 1.0),
               "res4": (lambda D: att_model(D, layer_timesteps=(1, 1, 1, 2), residual_connections={"3": [0, 1, 2, 3]}), 1.0)}
    for name, (mk, keep) in crosses.items():
        for D in (36, 132):
            for where, env in (("local", {}), ("global", FORCE_GLOBAL)):
                plan = (ATT_CUDNN_LOCAL if where == "local" else ATT_CUDNN_GLOBAL) if name == "cudnn" else (ATT_LOCAL if where == "local" else ATT_GLOBAL)
                out.append(Case("%s-%s-D%d" % (name, where, D), mk(D), "hubs", "mild", env, plan, "feature crosses", state_keep=keep))
    return out


CASES = {c.name: c for c in _cases()}

# the ABI checks (partial requests, prefilled buffers, bit identity) run on these
ABI_CASES = ["hubs-local-D36", "hubs-global-D132", "self_dup-local-D132"]

# the default-size batch: about 100 k nodes of synthetic molecules with hubs after them, hidden 100, two timesteps (float64 autograd of
# it on the CPU takes seconds per step)
DEFAULT_SIZE_MOLECULES = 5400
DEFAULT_SIZE_PARAMS = att_model(100, layer_timesteps=(2,), residual_connections={})


@functools.lru_cache(maxsize=None)
def default_size_batch():
    mols = synthetic.make_molecules(DEFAULT_SIZE_MOLECULES, seed=12)
    b = packing.pack_sparse_batch(packing.process_raw_graphs_sparse(mols), 8, 4)
    adj, indeg = b["adjacency_lists"], b["num_incoming_edges_per_type"]
    hadj, hindeg, _ = batch("hubs")
    V = indeg.shape[0]
    adj = [np.concatenate([np.asarray(a, np.int32).reshape(-1, 2), (h + V).astype(np.int32)]) for a, h in zip(adj, hadj)]
    return adj, np.concatenate([np.asarray(indeg, np.float32), hindeg])


def plan_matches(plan, pattern):
    return re.search(pattern, plan) is not None


def host_plan(params, T, adj, indeg, env, monkeypatch):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_FFMA_VARIANT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return PreparedGraph.host_only(params, T, adj, indeg, precision="fp32", num_sms=NUM_SMS, save_for_backward=True).info()["plan"]


# ---------------------------------------------------------------------------------------------------------------- tests
def test_batches_have_the_shapes_the_cases_claim():
    adj, indeg, T = batch("hubs")
    deg = indeg.sum(1)
    assert np.sum(deg == 0) >= 2
    for k in HUB_DEGREES:
        hits = np.flatnonzero(deg == k)
        assert hits.size, k
        if k > 1:
            assert any((indeg[v] > 0).sum() >= 3 for v in hits), k
    src, tgt, typ = O.message_arrays(adj)
    v300 = int(np.flatnonzero(deg == 300)[0])
    assert len(set(src[tgt == v300].tolist())) <= 20          # 300 messages through duplicate edges
    # big_hub: one component of more than 1000 nodes (no cut before node 1001), in-degree >= 1000
    adj, indeg, T = batch("big_hub")
    assert indeg.sum(1).max() >= 1000
    src, tgt, _ = O.message_arrays(adj)
    reach = np.zeros(indeg.shape[0], np.int64)
    np.maximum.at(reach, np.minimum(src, tgt), np.maximum(src, tgt))
    assert np.all(np.maximum.accumulate(reach)[:BIG_HUB_DEGREE] >= np.arange(1, BIG_HUB_DEGREE + 1))
    # self_dup
    adj, indeg, T = batch("self_dup")
    src, tgt, typ = O.message_arrays(adj)
    msgs = list(zip(src.tolist(), tgt.tolist(), typ.tolist()))
    into = lambda v: [m for m in msgs if m[1] == v]
    assert [m[:2] for m in into(SELF_ONLY)] == [(SELF_ONLY, SELF_ONLY)]
    assert (SELF_PLUS, SELF_PLUS) in [m[:2] for m in into(SELF_PLUS)] and len(into(SELF_PLUS)) >= 3
    assert sum(m == (8, DUP_TGT, 1) for m in msgs) == 2
    assert {m[2] for m in msgs if m[:2] == (12, TWO_TYPES_TGT)} == {0, 2}
    assert sum(s == d for s, d, _ in msgs) >= 20
    assert np.sum(indeg.sum(1) == 0) >= 2
    # t16_all: every type, one target with all 16; t16_ends: only 0 and 15; t1
    adj, indeg, T = batch("t16_all")
    assert T == 16 and all(a.shape[0] > 0 for a in adj) and ((indeg > 0).sum(1) == 16).any()
    adj, indeg, T = batch("t16_ends")
    assert T == 16 and [t for t in range(16) if adj[t].shape[0]] == [0, 15]
    adj, indeg, T = batch("t1")
    assert T == 1 and adj[0].shape[0] > 0


@pytest.mark.parametrize("D", [36, 256])
def test_score_regimes_reach_their_extremes(D):
    """In float64 at step 0: ``large`` has a score >= 90 (fp32 exp of it is inf), ``negative`` a node with >= 2 messages whose scores are
    all <= -90 (fp32 exp of each is below 1e-38, so their unshifted sum would be about 0, not about 1), ``mild`` stays small, and the
    a_t regimes have the weights they claim."""
    adj, indeg, T = batch("hubs")
    V = indeg.shape[0]
    p = att_model(D)
    for regime in REGIMES:
        h0 = regime_h0(regime, V, D)
        a = regime_weights(p, T, regime)[0]["edge_type_attention_weights"]
        sc, tgt = step0_scores(h0, adj, a)
        if regime == "large":
            assert sc.max() >= BOUND
            with np.errstate(over="ignore"):
                assert np.isinf(np.exp(np.float32(sc.max())))
        elif regime == "negative":
            nodes = [v for v in np.unique(tgt) if np.sum(tgt == v) >= 2 and sc[tgt == v].max() <= -BOUND]
            assert nodes
            with np.errstate(under="ignore"):
                assert np.sum(np.exp(sc[tgt == nodes[0]].astype(np.float32))) < 1e-38
        else:
            assert np.abs(sc).max() < 30
        if regime == "a_zero":
            assert a[1] == 0 and np.all(a[[0, 2, 3]] > 0)
        if regime == "a_negative":
            assert a[0] < 0 and a[2] < 0 and a[1] > 0


def _oracle_agree(adj, indeg, T, regime, p):
    import torch
    from oracle import c_oracle as CO
    V = indeg.shape[0]
    D = p["hidden_size"]
    h0 = regime_h0(regime, V, D)
    w = regime_weights(p, T, regime)
    vec = O.sparse_propagation_np(h0, adj, indeg, w, p, dtype=np.float64)
    scale = np.max(np.abs(vec))
    tor = O.sparse_propagation_torch(h0, adj, indeg, w, p, dtype=torch.float64).numpy()
    assert np.max(np.abs(tor - vec)) / scale < 1e-12
    if sum(a.shape[0] for a in adj) <= 3000:     # the loops restate every message in Python
        loops = O.sparse_propagation_loops(h0, adj, indeg, w, p)
        assert np.max(np.abs(loops - vec)) / scale < 1e-12
    if os.path.exists(CO.LIB):                  # built by build()
        c = CO.sparse_propagation_c(h0, adj, indeg, w, p)
        assert np.max(np.abs(c - vec)) / scale < 1e-12
    assert np.all(np.isfinite(vec))


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_oracle_statements_agree_on_every_kind(kind):
    adj, indeg, T = batch(kind)
    _oracle_agree(adj, indeg, T, "mild", att_model(8))


@pytest.mark.parametrize("regime", REGIMES[1:])
def test_oracle_statements_agree_on_every_regime(regime):
    adj, indeg, T = batch("hubs")
    _oracle_agree(adj, indeg, T, regime, att_model(8, layer_timesteps=(2,), residual_connections={}))


@pytest.mark.parametrize("cell", ["CudnnCompatibleGRUCell", "RNN"])
def test_oracle_statements_agree_on_the_crossed_cells(cell):
    adj, indeg, T = batch("self_dup")
    _oracle_agree(adj, indeg, T, "mild", att_model(8, cell=cell))


@pytest.mark.parametrize("case", sorted(CASES), ids=str)
def test_case_reaches_its_plan(case, monkeypatch):
    c = CASES[case]
    adj, indeg, T = batch(c.kind)
    plan = host_plan(c.params, T, adj, indeg, c.env, monkeypatch)
    assert plan_matches(plan, c.plan), (c.plan, plan)


def test_default_size_batch_reaches_a_local_plan(monkeypatch):
    adj, indeg = default_size_batch()
    assert 95000 <= indeg.shape[0] <= 110000
    assert indeg.sum(1).max() == 300
    plan = host_plan(DEFAULT_SIZE_PARAMS, 4, adj, indeg, {}, monkeypatch)
    assert plan_matches(plan, ATT_LOCAL), plan


def test_seventeen_edge_types_with_attention_are_refused():
    """At most 16 edge types with attention (the target backward sums d a_t in a 16-slot shared array).  The model shape check refuses
    17, both where an engine is created and where a batch is prepared without one; 16 is accepted."""
    from gated_graph_neural_network_samples_b200.engine import GgnnError, PreparedGraph, PropagationEngine
    adj, indeg = component_graph(17, V_target=60, seed=2)
    with pytest.raises(GgnnError, match="propagation attention supports at most 16 edge types"):
        PropagationEngine(att_model(8), 17)          # refused by the shape check, before any device is touched
    with pytest.raises(GgnnError, match="propagation attention supports at most 16 edge types"):
        PreparedGraph.host_only(att_model(8), 17, adj, indeg, num_sms=NUM_SMS)
    adj, indeg, T = batch("t16_all")
    assert "+attention" in PreparedGraph.host_only(att_model(8), 16, adj, indeg, num_sms=NUM_SMS).info()["plan"]
