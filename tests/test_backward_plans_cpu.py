"""CPU: the cases of tests/test_gpu_backward_plans.py, pinned to the forward plan they are meant to reach, and the float64 oracle on the
model shapes those cases add.

The gradient tests there are only as good as the plan each case lands on: the backward reads the activations the forward kernel saved,
and every plan writes them with its own code.  Here every sparse, binary-dense and GCN case is built through the host-only prepare calls
at 132 SMs (an H100 SXM) with the same environment settings, and the plan text must be the one the GPU test expects.  A later change to
the planner that moves a case onto another kernel fails here, without a GPU.  (The weighted dense cases cannot be pinned here: the
host-only dense prepare refuses weighted matrices.  The GPU test checks their plan on the device.)
"""
import functools
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from oracle import ggnn_oracle as O
from tests import _util as U
from tests import gcn_oracle as G

NUM_SMS = 132

# ---------------------------------------------------------------------------------------------------------------- plan texts
FFMA_LOCAL_64 = r"^fp32-ffma LOCAL\(.* rows/tile<=64 warps=8 colsplit=1 "      # variant 0
FFMA_LOCAL_32 = r"^fp32-ffma LOCAL\(.* rows/tile<=32 warps=8 colsplit=2 "      # variant 1
FFMA_GLOBAL = r"^fp32-ffma GLOBAL\("
FFMA_CUDNN_LOCAL = r"^fp32-ffma\+cudnn-gru LOCAL\("
FFMA_CUDNN_GLOBAL = r"^fp32-ffma\+cudnn-gru GLOBAL\("
FFMA_ATT_GLOBAL = r"^fp32-ffma\+attention GLOBAL\("
TC_LOCAL_64 = r"^wgmma-bf16x3 LOCAL\(.* \(compact 64-row operand tiles\) "
TC_LOCAL_128 = r"^wgmma-bf16x3 LOCAL\(.* rows/tile<=128 DP="                    # no "compact": 128-row operand tiles
TC_GLOBAL = r"^wgmma-bf16x3 GLOBAL\(.* rows/tile<=128 DP="
TC_STREAM = r"^wgmma-bf16x3 STREAM\("
GCN_TC_LOCAL = r"^gcn-wgmma-bf16x3 LOCAL\("
GCN_TC_GLOBAL = r"^gcn-wgmma-bf16x3 GLOBAL\("
GCN_FFMA = r"^gcn-fp32-ffma GLOBAL\("

FORCE_GLOBAL = {"GGNN_FORCE_GLOBAL": "1"}
FORCE_STREAM = {"GGNN_TC_STREAM": "1"}


def model(cell, D, layer_timesteps=(2, 1), residual_connections=None, act="ReLU", bias=True, avg=False, attention=False):
    return {"hidden_size": D, "layer_timesteps": list(layer_timesteps),
            "residual_connections": {"1": [0]} if residual_connections is None else residual_connections,
            "use_edge_bias": bias, "use_edge_msg_avg_aggregation": avg, "graph_rnn_cell": cell, "graph_rnn_activation": act,
            "use_propagation_attention": attention}


# ---------------------------------------------------------------------------------------------------------------- batches
def component_graph(T, V_target=420, seed=0):
    """Small components whose edges (both directions) take types uniform over ``T``: two isolated nodes, a pair joined by one type-0
    edge (each of its nodes receives messages of a single type), then random trees with a few extra edges.  Every type occurs.
    Returns the reference wire format: per-type ``[E_t, 2]`` (source, target) int32 lists and the ``[V, T]`` in-degree table."""
    rng = np.random.default_rng(seed)
    und, off = [(2, 3)], 4            # nodes 0, 1 isolated; nodes 2 -- 3 the single-type pair
    while off < V_target:
        n = int(rng.integers(3, 20))
        und += [(off + int(rng.integers(0, i)), off + i) for i in range(1, n)]
        for _ in range(n // 4):
            a, b = rng.choice(n, 2, replace=False)
            und.append((off + int(a), off + int(b)))
        off += n
    types = rng.integers(0, T, len(und))
    types[0] = 0
    types[1:T + 1] = np.arange(T)     # every type occurs
    V = off
    adj = []
    for t in range(T):
        e = np.asarray([u for u, k in zip(und, types) if k == t], np.int32).reshape(-1, 2)
        adj.append(np.concatenate([e, e[:, ::-1]], axis=0).astype(np.int32))
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg


@functools.lru_cache(maxsize=None)
def _molecules(n, T, seed):
    mols = synthetic.make_molecules(n, seed=seed, num_bond_types=T)
    return packing.pack_sparse_batch(packing.process_raw_graphs_sparse(mols), 8, T)   # (h0 is drawn per hidden size below)


def sparse_batch(kind, D, T):
    """(adjacency lists, in-degree table, h0 [V, D] float32) of a batch kind: ``mol<n>`` = n synthetic molecules with T bond types,
    ``comp`` = ``component_graph(T)``."""
    if kind == "comp":
        adj, indeg = component_graph(T, seed=T)
        h0 = np.random.default_rng(100 + D).normal(0, 1, (indeg.shape[0], D)).astype(np.float32)
        return adj, indeg, h0
    b = _molecules(int(kind[3:]), T, 3)
    V = b["num_incoming_edges_per_type"].shape[0]
    h0 = np.random.default_rng(200 + D).normal(0, 1, (V, D)).astype(np.float32)
    return b["adjacency_lists"], b["num_incoming_edges_per_type"], h0


# ---------------------------------------------------------------------------------------------------------------- the GGNN cases
def smooth_on_tensor_cores(precision):
    """ReLU on the fp32 kernel, tanh on the bf16x3 plans.  ReLU's derivative jumps at 0: where a pre-activation lies within the forward's
    rounding of 0 (about 1e-5 relative on bf16x3, 5e-7 on fp32), the engine and float64 autograd take opposite sides of the jump and
    that node's gradient differs by O(1).  A 24-molecule batch at hidden 100 has about 10 pre-activations within 1e-5 of the largest,
    1024 molecules have hundreds; with ReLU the bf16x3 plans measured 1e-2 to 7e-2 on d h0 there, the same number on three different
    kernels for the same batch.  That is the activation's conditioning, not a kernel error, so the tensor-core cases use tanh."""
    return "ReLU" if precision == "fp32" else "tanh"


class Case:
    def __init__(self, name, params, T, batch, precision, env, plan):
        self.name, self.params, self.T, self.batch, self.precision, self.env, self.plan = name, params, T, batch, precision, env, plan

    def __repr__(self):
        return self.name


def _plan_matrix():
    plans = [   # (plan id, precision, env, batch, hidden sizes, plan text)
        ("ffma0-local", "fp32", {"GGNN_FFMA_VARIANT": "0"}, "mol24", (36, 100), FFMA_LOCAL_64),
        ("ffma1-local", "fp32", {"GGNN_FFMA_VARIANT": "1"}, "mol24", (36, 100), FFMA_LOCAL_32),
        ("ffma-global", "fp32", FORCE_GLOBAL, "mol24", (100, 252), FFMA_GLOBAL),
        ("tc-local64", "bf16x3", {}, "mol24", (20, 100), TC_LOCAL_64),
        ("tc-local128", "bf16x3", {}, "mol1024", (100,), TC_LOCAL_128),
        ("tc-global", "bf16x3", FORCE_GLOBAL, "mol24", (20, 100, 128), TC_GLOBAL),
        ("stream-forced", "bf16x3", FORCE_STREAM, "mol24", (20, 100), TC_STREAM),
        ("stream", "bf16x3", {}, "mol24", (132, 204, 256), TC_STREAM),
    ]
    out = []
    for pid, prec, env, batch, Ds, plan in plans:
        for D in Ds:
            for cell in ("GRU", "RNN"):
                out.append(Case("%s-%s-D%d" % (pid, cell.lower(), D), model(cell, D, act=smooth_on_tensor_cores(prec)), 4, batch, prec, env, plan))
    cudnn = lambda D: model("CudnnCompatibleGRUCell", D, act="tanh")
    out += [Case("ffma-local-cudnn-D100", cudnn(100), 4, "mol24", "fp32", {}, FFMA_CUDNN_LOCAL),
            Case("ffma-global-cudnn-D100", cudnn(100), 4, "mol24", "fp32", FORCE_GLOBAL, FFMA_CUDNN_GLOBAL),
            Case("ffma-global-attention-D36", model("GRU", 36, act="tanh", attention=True), 4, "mol24", "fp32", FORCE_GLOBAL, FFMA_ATT_GLOBAL)]
    return out


def _edge_shapes():
    """Shapes at the backward kernels' edges, on the fp32 kernel and on one tensor-core plan each.
    T = 1, 3: the edge-bias gradient's scalar loads (T not a multiple of 4); T = 17, 32: the edge-weight gradient split into 16-type
    launches, and the tile-local kernel without its shared-memory CSR cache.  All with avg aggregation over components that include
    isolated nodes and nodes whose messages have a single type."""
    out = []
    tc = {1: ("stream-forced", FORCE_STREAM, TC_STREAM), 3: ("tc-global", FORCE_GLOBAL, TC_GLOBAL), 17: ("tc-local64", {}, TC_LOCAL_64),
          32: ("tc-local64", {}, TC_LOCAL_64)}
    for T in (1, 3, 17, 32):
        p = model("GRU", 36, act="tanh", avg=True)
        out.append(Case("T%d-ffma-D36" % T, p, T, "comp", "fp32", {}, r"^fp32-ffma LOCAL\("))
        pid, env, plan = tc[T]
        out.append(Case("T%d-%s-D20" % (T, pid), dict(p, hidden_size=20), T, "comp", "bf16x3", env, plan))
    # four residual inputs into the last layer, one of them the layer's own input (r == l)
    res4 = lambda D: model("GRU", D, layer_timesteps=(1, 1, 1, 2), residual_connections={"3": [0, 1, 2, 3]}, act="tanh", avg=True)
    out += [Case("res4-ffma-D36", res4(36), 4, "mol24", "fp32", {}, r"^fp32-ffma LOCAL\("),
            Case("res4-stream-forced-D20", res4(20), 4, "mol24", "bf16x3", FORCE_STREAM, TC_STREAM)]
    # a layer of zero steps, read by the next layer through a residual (its input and its output: the same state)
    zero = lambda D, cell, prec: model(cell, D, layer_timesteps=(2, 0, 1), residual_connections={"2": [1, 2]}, act=smooth_on_tensor_cores(prec))
    out += [Case("zero-step-ffma-%s-D36" % c.lower(), zero(36, c, "fp32"), 4, "mol24", "fp32", {}, r"^fp32-ffma LOCAL\(") for c in ("GRU", "RNN")]
    out += [Case("zero-step-tc-local64-%s-D20" % c.lower(), zero(20, c, "bf16x3"), 4, "mol24", "bf16x3", {}, TC_LOCAL_64) for c in ("GRU", "RNN")]
    return out


PLAN_MATRIX = _plan_matrix()
EDGE_SHAPES = _edge_shapes()
SPARSE_CASES = {c.name: c for c in PLAN_MATRIX + EDGE_SHAPES}

# partial requests and determinism run on a few of the cases above
PARTIAL_CASES = ["ffma1-local-gru-D36", "ffma1-local-rnn-D36", "ffma-local-cudnn-D100", "tc-local64-gru-D20"]
DETERMINISM_CASES = ["tc-local64-gru-D100", "tc-global-rnn-D100", "stream-gru-D132", "ffma0-local-gru-D100"]

# dense: (name, precision, hidden, weighted, plan text).  Every case goes through the CSR builder; the weighted ones with slot weights.
DENSE_CASES = [("weighted-fp32-D24", "fp32", 24, True, r"^fp32-ffma LOCAL\("),
               ("weighted-tc-D100", "bf16x3", 100, True, TC_LOCAL_64),
               ("binary-tc-D100", "bf16x3", 100, False, TC_LOCAL_64)]
DENSE_T, DENSE_STEPS, DENSE_V = 4, 3, 29


def dense_batch(D, weighted):
    mols = synthetic.make_molecules(10, seed=8)
    db = packing.pack_dense_batch(mols, DENSE_V, D, DENSE_T)
    rng = np.random.default_rng(2)
    A = np.asarray(db["adjacency_matrix"], np.float32)
    if weighted:
        A = (A * rng.uniform(0.25, 1.75, A.shape)).astype(np.float32)
    h0 = (db["initial_node_representation"] + rng.normal(0, 0.1, db["initial_node_representation"].shape)).astype(np.float32)
    return A, h0


def dense_params(D):
    return U.dense_params_as_engine_params({"num_timesteps": DENSE_STEPS, "use_edge_bias": True}, D)


# GCN: (name, precision, hidden, graph kind, keep, env, plan text)
GCN_CASES = ([("local-D%d-keep%s" % (D, k), "bf16x3", D, "components", k, {}, GCN_TC_LOCAL) for D in (12, 100, 128) for k in (1.0, 0.8)]
             + [("ffma-D%d" % D, "fp32", D, "components", 1.0, {}, GCN_FFMA) for D in (132, 256)]
             + [("global-D128", "bf16x3", 128, "random", 1.0, {}, GCN_TC_GLOBAL)])
GCN_LAYERS = 3


def gcn_batch(D, kind, seed=0):
    """(V, [nnz, 2] list, [nnz] weights, kernels, biases, h0)."""
    rng = np.random.default_rng(seed + D)
    if kind == "components":
        V, lst, w = G.component_list(list(rng.integers(3, 30, 40)), rng)
    else:
        V = 300
        lst, w = G.random_gcn_list(V, 2000, rng, isolated=(0, 7))
    ks = [G.glorot((D, D), rng) for _ in range(GCN_LAYERS)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(GCN_LAYERS)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    return V, lst, w, ks, bs, h0


def plan_matches(plan, pattern):
    return re.search(pattern, plan) is not None


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("case", sorted(SPARSE_CASES), ids=str)
def test_sparse_case_reaches_its_plan(case, monkeypatch):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    c = SPARSE_CASES[case]
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    adj, indeg, _ = sparse_batch(c.batch, c.params["hidden_size"], c.T)
    plan = PreparedGraph.host_only(c.params, c.T, adj, indeg, precision=c.precision, num_sms=NUM_SMS, save_for_backward=True).info()["plan"]
    assert plan_matches(plan, c.plan), (c.plan, plan)


@pytest.mark.parametrize("name,precision,D,weighted,pattern", [c for c in DENSE_CASES if not c[3]], ids=lambda x: str(x))
def test_binary_dense_case_reaches_its_plan(name, precision, D, weighted, pattern):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    A, _ = dense_batch(D, weighted)
    plan = PreparedGraph.host_only_dense(dense_params(D), DENSE_T, A, precision=precision, num_sms=NUM_SMS, save_for_backward=True).info()["plan"]
    assert plan_matches(plan, pattern), (pattern, plan)


@pytest.mark.parametrize("name,precision,D,kind,keep,env,pattern", GCN_CASES, ids=[c[0] for c in GCN_CASES])
def test_gcn_case_reaches_its_plan(name, precision, D, kind, keep, env, pattern, monkeypatch):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    V, lst, w, _, _, _ = gcn_batch(D, kind)
    plan = PreparedGraph.host_only_gcn(D, GCN_LAYERS, V, lst, w, use_bias=True, precision=precision, num_sms=NUM_SMS,
                                       save_for_backward=True).info()["plan"]
    assert plan_matches(plan, pattern), (pattern, plan)


def test_batches_have_the_shapes_the_cases_claim():
    """The 128-row LOCAL case has more tiles than the chip has SMs; the component graphs have isolated nodes, nodes with messages of a
    single type, and every edge type."""
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    c = SPARSE_CASES["tc-local128-gru-D100"]
    adj, indeg, _ = sparse_batch(c.batch, 100, 4)
    assert PreparedGraph.host_only(c.params, 4, adj, indeg, precision="bf16x3", num_sms=NUM_SMS).info()["num_tiles"] > NUM_SMS
    for T in (1, 3, 17, 32):
        adj, indeg = component_graph(T, seed=T)
        assert all(a.shape[0] > 0 for a in adj)
        deg = indeg.sum(1)
        assert np.sum(deg == 0) >= 2
        single = (deg > 0) & ((indeg > 0).sum(1) == 1)
        assert single[2] and single[3]


# the model shapes the GPU cases add, on which the three oracle statements must agree before the engine is blamed for a difference
ORACLE_SHAPES = {
    "T17_avg_bias": (model("GRU", 8, act="tanh", avg=True), 17),
    "T32_rnn_relu": (model("RNN", 8), 32),
    "res4_self": (model("GRU", 8, layer_timesteps=(1, 1, 1, 2), residual_connections={"3": [0, 1, 2, 3]}, act="tanh", avg=True), 4),
    "zero_step": (model("RNN", 8, layer_timesteps=(2, 0, 1), residual_connections={"2": [1, 2]}), 4),
    "zero_step_gru": (model("GRU", 8, layer_timesteps=(2, 0, 1), residual_connections={"2": [1, 2]}), 4),
}


@pytest.mark.parametrize("name", sorted(ORACLE_SHAPES))
def test_oracle_statements_agree_on_the_new_shapes(name):
    import torch
    p, T = ORACLE_SHAPES[name]
    adj, indeg = component_graph(T, V_target=60, seed=T + 1)
    h0 = np.random.default_rng(4).normal(0, 1, (indeg.shape[0], 8))
    w = O.init_sparse_weights(p, T, np.random.default_rng(5))
    loops = O.sparse_propagation_loops(h0, adj, indeg, w, p, dtype=np.float64, return_all_layers=True)
    vec = O.sparse_propagation_np(h0, adj, indeg, w, p, dtype=np.float64, return_all_layers=True)
    tor = O.sparse_propagation_torch(h0, adj, indeg, w, p, dtype=torch.float64, return_all_layers=True)
    assert len(loops) == len(vec) == len(tor) == len(p["layer_timesteps"]) + 1
    for l, (a, b, c) in enumerate(zip(loops, vec, tor)):
        scale = max(np.max(np.abs(a)), 1e-30)
        assert np.max(np.abs(a - b)) / scale < 1e-12, l
        assert np.max(np.abs(a - c.numpy())) / scale < 1e-12, l
    if p["layer_timesteps"][1] == 0:
        np.testing.assert_array_equal(loops[1], loops[2])
