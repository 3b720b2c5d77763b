"""CPU: the batch scripts of tests/test_gpu_engine_lifetime.py and tests/test_gpu_training_steps.py, pinned to the plans they claim.

One engine serves every batch of a training run, and each batch may change the node count, the plan, the save flag, the dropout seed
and the weights.  The GPU tests run scripted sequences of such batches through ONE engine; a sequence is only worth as much as the
transitions it really makes.  Here every scripted batch is prepared through the host-only calls at 132 SMs (an H100 SXM) with the
step's environment, and must reach the plan its step names; each script must grow V and then shrink it below an earlier maximum; the
hub batch must carry virtual rows with more than 7 messages; and the training dataset's batches must span at least two plans.  A
change to the plan heuristics that turns a sequence into "all LOCAL" fails here, without a GPU.
"""
import functools
import re
import zlib

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from tests import gcn_oracle as G
from tests.test_backward_plans_cpu import NUM_SMS, component_graph, sparse_batch

FORCE_GLOBAL = {"GGNN_FORCE_GLOBAL": "1"}


# ---------------------------------------------------------------------------------------------------------------- plan texts
def tc(prec, kind):
    """Plan text of the tile-local wgmma (compact / 128-row LOCAL, GLOBAL) or streaming plan at bf16x3 or bf16."""
    return {"local64": r"^wgmma-%s LOCAL\(.* \(compact 64-row operand tiles\) ",
            "local128": r"^wgmma-%s LOCAL\(.* rows/tile<=128 DP=",
            "global": r"^wgmma-%s GLOBAL\(.* rows/tile<=128 DP=",
            "stream": r"^wgmma-%s STREAM\("}[kind] % prec


FFMA = {"v0": r"^fp32-ffma LOCAL\(.* rows/tile<=64 warps=8 colsplit=1 ", "v1": r"^fp32-ffma LOCAL\(.* rows/tile<=32 warps=8 colsplit=2 ",
        "global": r"^fp32-ffma GLOBAL\(", "any": r"^fp32-ffma[ (]"}


def plan_of(precision, kind):
    return FFMA[kind] if precision == "fp32" else tc(precision, kind)


# ---------------------------------------------------------------------------------------------------------------- models
# the reference's default sparse model (chem_tensorflow_sparse.py:43-60) with edge bias: the residuals make the offsets of the layer
# states in the engine's state buffer depend on V
DEFAULT = {"hidden_size": 100, "layer_timesteps": [2, 2, 1, 2, 1], "residual_connections": {"2": [0], "4": [0, 2]}, "use_edge_bias": True,
           "use_edge_msg_avg_aggregation": True, "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}
ATTENTION = dict(DEFAULT, hidden_size=36, layer_timesteps=[2, 1], residual_connections={"1": [0]}, use_propagation_attention=True)
CUDNN = dict(DEFAULT, hidden_size=36, layer_timesteps=[2, 1], residual_connections={"1": [0]}, graph_rnn_cell="CudnnCompatibleGRUCell")
# BASELINE config 4's shape: hidden 256, 8 edge types, always the streaming plan
CFG4 = {"hidden_size": 256, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "use_edge_bias": True,
        "use_edge_msg_avg_aggregation": False, "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}


# ---------------------------------------------------------------------------------------------------------------- batches
def _pack(mols, T):
    b = packing.pack_sparse_batch(packing.process_raw_graphs_sparse(mols), 8, T)
    return b["adjacency_lists"], b["num_incoming_edges_per_type"]


def hub_graph(V, hubs, T, seed):
    """``hubs`` targets that each receive 9 .. 40 messages of one type (virtual rows whose source list runs past the 7 inline entries),
    the other nodes a few random messages each."""
    rng = np.random.default_rng(seed)
    lists = [[] for _ in range(T)]
    for h in range(hubs):
        tgt = int(rng.integers(0, V))
        lists[h % T] += [(int(s), tgt) for s in rng.integers(0, V, int(rng.integers(9, 41)))]
    for tgt in range(V):
        for _ in range(int(rng.integers(0, 3))):
            lists[int(rng.integers(0, T))].append((int(rng.integers(0, V)), tgt))
    adj = [np.asarray(sorted(e), np.int32).reshape(-1, 2) for e in lists]
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg


@functools.lru_cache(maxsize=None)
def _graph(kind, T):
    """(adjacency lists, [V, T] in-degrees) of a batch kind:
    ``mol<n>``        n synthetic molecules (tests/test_backward_plans_cpu.py's batches)
    ``mol<n>+<m>``    n molecules and one m-node molecule (a component larger than any tile)
    ``empty``         V = 0;  ``single``: one isolated node
    ``hub<V>x<h>``    hub_graph(V, h)
    ``comp``          component_graph(T)"""
    if kind == "empty":
        return [np.zeros((0, 2), np.int32) for _ in range(T)], np.zeros((0, T), np.float32)
    if kind == "single":
        return [np.zeros((0, 2), np.int32) for _ in range(T)], np.zeros((1, T), np.float32)
    if kind == "comp":
        return component_graph(T, seed=T)
    m = re.fullmatch(r"hub(\d+)x(\d+)", kind)
    if m:
        return hub_graph(int(m.group(1)), int(m.group(2)), T, seed=int(m.group(1)))
    m = re.fullmatch(r"mol(\d+)\+(\d+)", kind)
    if m:
        n, big = int(m.group(1)), int(m.group(2))
        mols = synthetic.make_molecules(n, seed=5, num_bond_types=T)
        mols.append(synthetic.make_molecule(np.random.default_rng(6), min_atoms=big, max_atoms=big, mean_atoms=big))
        return _pack(mols, T)
    if T == 4:
        adj, indeg, _ = sparse_batch(kind, 8, T)
        return adj, indeg
    return _pack(synthetic.make_molecules(int(kind[3:]), seed=3, num_bond_types=T), T)


def batch(kind, D, T, seed=0):
    """(adjacency lists, in-degrees, h0 [V, D] float32); h0 is drawn per (kind, D, seed)."""
    adj, indeg = _graph(kind, T)
    rng = np.random.default_rng(zlib.crc32(("%s/%d/%d" % (kind, D, seed)).encode()))
    return adj, indeg, rng.normal(0, 1, (indeg.shape[0], D)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------- scripts
class Step:
    """One batch of a sequence: the batch kind, the weights to bind first (an int seed; None keeps the bound ones), save_for_backward,
    the state keep probability and dropout seed, the environment while the batch is prepared, and the plan it must reach."""

    def __init__(self, kind, weights, save, keep, seed, plan, env=None):
        self.kind, self.weights, self.save, self.keep, self.seed, self.plan, self.env = kind, weights, save, keep, seed, plan, env or {}

    def __repr__(self):
        return "%s(w=%s save=%d keep=%g)" % (self.kind, self.weights, self.save, self.keep)


def ggnn_script(precision, short=False):
    """The default model's sequence: compact LOCAL -> 128-row LOCAL (V grows, the state and save buffers grow, new weights) -> the big
    component (STREAM on the tensor-core precisions, GLOBAL on fp32) -> step 1's batch again under GGNN_FORCE_GLOBAL with the weights
    unchanged -> empty -> a single node -> 5 molecules without save (validation) -> step 2's batch with step 2's weights bound again."""
    p = lambda kind: plan_of(precision, kind)
    local_small, local_big = ("v1", "v0") if precision == "fp32" else ("local64", "local128")
    big = "global" if precision == "fp32" else "stream"
    steps = [Step("mol24", 1, True, 0.9, 11, p(local_small)),
             Step("mol1024", 2, True, 1.0, 0, p(local_big)),
             Step("mol40+300", None, True, 0.9, 12, p(big)),
             Step("mol24", None, True, 1.0, 0, p("global"), FORCE_GLOBAL),
             Step("empty", None, True, 1.0, 0, None),
             Step("single", 4, True, 0.9, 13, None),
             Step("mol5", None, False, 1.0, 0, p(local_small)),
             Step("mol1024", 2, True, 1.0, 0, p(local_big))]
    if short:   # the plan switches without the empty / single-node steps
        steps = [steps[i] for i in (0, 1, 2, 3, 6)]
    return steps


def small_model_script(precision, attention):
    """Attention: att_buf holds [steps][M] probabilities when saving, [M] otherwise: save off at a small M, save on at a larger M, then
    save off at a small M again.  Both models run on the fp32 kernel at every precision."""
    plan = r"^fp32-ffma\+%s (LOCAL|GLOBAL)\(" % ("attention" if attention else "cudnn-gru")
    return [Step("mol24", 1, False, 1.0, 0, plan), Step("mol1024", 2, True, 0.9, 21, plan), Step("mol5", None, False, 1.0, 0, plan),
            Step("mol40+300", 3, True, 1.0, 0, plan)]


def cfg4_script():
    """Hidden 256, 8 edge types: always STREAM.  V grows and shrinks; a batch with hub nodes is followed by one with none, then one with
    fewer hubs; save toggles."""
    s = tc("bf16x3", "stream")
    return [Step("mol20", 1, True, 1.0, 0, s), Step("hub900x12", None, False, 1.0, 0, s), Step("mol80", 2, True, 0.9, 31, s),
            Step("hub300x3", None, False, 1.0, 0, s), Step("mol10", None, True, 1.0, 0, s)]


# GCN: (graph kind, weights seed, save, keep, dropout seed, plan by precision); "big" holds a 200-node component: more than a tile
GCN_D, GCN_L = 100, 3
GCN_PLANS = {"bf16x3": {"local": r"^gcn-wgmma-bf16x3 LOCAL\(", "global": r"^gcn-wgmma-bf16x3 GLOBAL\("},
             "fp32": {"local": r"^gcn-fp32-ffma ", "global": r"^gcn-fp32-ffma "}}
GCN_SCRIPT = [("small", 1, True, 0.8, 41, "local"), ("big", 2, False, 1.0, 0, "global"), ("big", 3, True, 0.9, 42, "global"),
              ("empty", 4, True, 1.0, 0, None), ("small", 5, False, 0.8, 43, "local"), ("medium", 6, True, 1.0, 0, "local")]


@functools.lru_cache(maxsize=None)
def gcn_graph(kind):
    """(V, [nnz, 2] list, [nnz] weights) of a GCN batch kind."""
    rng = np.random.default_rng({"small": 1, "big": 2, "medium": 3, "empty": 4}[kind])
    if kind == "empty":
        return 0, np.zeros((0, 2), np.int64), np.zeros(0, np.float32)
    sizes = {"small": list(rng.integers(3, 30, 20)), "medium": list(rng.integers(3, 30, 60)), "big": list(rng.integers(3, 30, 30)) + [200]}[kind]
    return G.component_list(sizes, rng)


# dense: (weighted, b, v); binary matrices go through the CSR builder, weighted ones walk the matrix
DENSE_T, DENSE_STEPS = 4, 3
DENSE_SCRIPT = [(False, 10, 29), (True, 16, 24), (False, 24, 29), (True, 6, 20), (False, 8, 12)]


def dense_matrix(weighted, b, v, seed=0):
    mols = synthetic.make_molecules(b, seed=8 + b)
    db = packing.pack_dense_batch(mols, v, 8, DENSE_T) if all(len(m["node_features"]) <= v for m in mols) else None
    if db is None:   # molecules larger than v: clip to v atoms
        mols = synthetic.make_molecules(b, seed=8 + b, max_atoms=v)
        db = packing.pack_dense_batch(mols, v, 8, DENSE_T)
    A = np.asarray(db["adjacency_matrix"], np.float32)
    if weighted:
        A = (A * np.random.default_rng(seed + b).uniform(0.25, 1.75, A.shape)).astype(np.float32)
    return A


# ---------------------------------------------------------------------------------------------------------------- the training dataset
def training_molecules(n=80, seed=4, T=4):
    """Synthetic molecules plus two raw graphs of 200+ nodes in the reference JSON schema, two tasks."""
    mols = synthetic.make_molecules(n, seed=seed, num_bond_types=T)
    rng = np.random.default_rng(seed + 1)
    mols[7:7] = [synthetic.make_molecule(rng, min_atoms=200, max_atoms=260, mean_atoms=230) for _ in range(2)]
    return [dict(m, targets=[m["targets"][0], [float(rng.normal())]]) for m in mols]


# the sparse plug-in's model in tests/test_gpu_training_steps.py: several batches per epoch, and the ones holding a 200+-node graph leave
# the tile-local plans
TRAIN_MODEL = {"hidden_size": 32, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "use_edge_bias": True,
               "use_edge_msg_avg_aggregation": True, "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh", "batch_size": 300}


# ---------------------------------------------------------------------------------------------------------------- tests
def _host_plan(params, T, kind, precision, env, monkeypatch, save=True):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    adj, indeg = _graph(kind, T)
    g = PreparedGraph.host_only(params, T, adj, indeg, precision=precision, num_sms=NUM_SMS, save_for_backward=save)
    return g


SCRIPTS = {"ggnn-bf16x3": (DEFAULT, 4, "bf16x3", ggnn_script("bf16x3")), "ggnn-fp32": (DEFAULT, 4, "fp32", ggnn_script("fp32")),
           "ggnn-bf16": (DEFAULT, 4, "bf16", ggnn_script("bf16", short=True)),
           "attention": (ATTENTION, 4, "bf16x3", small_model_script("bf16x3", True)), "cudnn": (CUDNN, 4, "fp32", small_model_script("fp32", False)),
           "cfg4": (CFG4, 8, "bf16x3", cfg4_script())}


@pytest.mark.parametrize("name", sorted(SCRIPTS))
def test_every_scripted_batch_reaches_its_plan(name, monkeypatch):
    params, T, precision, steps = SCRIPTS[name]
    for i, s in enumerate(steps):
        info = _host_plan(params, T, s.kind, precision, s.env, monkeypatch, s.save).info()
        if s.plan is not None:
            assert re.search(s.plan, info["plan"]), (name, i, s, info["plan"])


@pytest.mark.parametrize("name", sorted(SCRIPTS))
def test_every_script_grows_and_then_shrinks_v(name):
    _, T, _, steps = SCRIPTS[name]
    Vs = [_graph(s.kind, T)[1].shape[0] for s in steps]
    grow = next(i for i in range(1, len(Vs)) if Vs[i] > Vs[i - 1])
    assert any(Vs[j] < max(Vs[:j]) for j in range(grow + 1, len(Vs))), Vs


def test_the_hub_batches_have_long_virtual_rows_and_the_molecules_none(monkeypatch):
    """hub900x12 has virtual rows with more than 7 messages (past vinfo's inline entries), mol80 has none that long, hub300x3 fewer."""
    long_rows = {}
    for kind in ("hub900x12", "mol80", "hub300x3"):
        g = _host_plan(CFG4, 8, kind, "bf16x3", {}, monkeypatch)
        a = g.arrays(8)
        cnt = np.diff(a["row_ptr"])
        long_rows[kind] = int(np.sum(cnt > 7))
        if kind.startswith("hub"):
            assert np.sum(a["pair_src"] <= -2) > 0, kind      # (target, type) pairs with several messages: virtual rows
    assert long_rows["hub900x12"] > long_rows["hub300x3"] > 0 == long_rows["mol80"], long_rows


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_every_gcn_batch_reaches_its_plan(precision):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    Vs = []
    for kind, _, save, _, _, plan in GCN_SCRIPT:
        V, lst, w = gcn_graph(kind)
        Vs.append(V)
        info = PreparedGraph.host_only_gcn(GCN_D, GCN_L, V, lst, w, use_bias=True, precision=precision, num_sms=NUM_SMS,
                                           save_for_backward=save).info()
        if plan is not None:
            assert re.search(GCN_PLANS[precision][plan], info["plan"]), (kind, info["plan"])
    assert max(Vs[:2]) > Vs[0] and Vs[-2] < max(Vs), Vs


def test_dense_script_alternates_binary_and_weighted_matrices():
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    from tests.test_backward_plans_cpu import dense_params
    for weighted, b, v in DENSE_SCRIPT:
        A = dense_matrix(weighted, b, v)
        assert A.shape == (b, DENSE_T, v, v)
        assert np.any((A != 0) & (A != 1)) == weighted
        if not weighted:
            plan = PreparedGraph.host_only_dense(dense_params(100), DENSE_T, A, precision="bf16x3", num_sms=NUM_SMS).info()["plan"]
            assert "binary dense adjacency -> CSR" in plan, plan


@pytest.mark.parametrize("precision,plans", [("bf16x3", {"LOCAL", "STREAM"}), ("fp32", {"LOCAL", "GLOBAL"})])
def test_training_batches_span_at_least_two_plans(precision, plans):
    """The training dataset, batched as the sparse plug-in batches it, at the model of tests/test_gpu_training_steps.py: the batches
    holding a 200+-node graph take STREAM on bf16x3 and GLOBAL on fp32, the others a tile-local plan."""
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    flat = packing.FlatSparseGraphs(packing.process_raw_graphs_sparse(training_molecules(), [0, 1]), 4)
    seen = []
    for b in flat.iter_minibatches(np.arange(flat.num_graphs), TRAIN_MODEL["batch_size"], TRAIN_MODEL["hidden_size"]):
        plan = PreparedGraph.host_only(TRAIN_MODEL, 4, b["adjacency_lists"], b["num_incoming_edges_per_type"], precision=precision,
                                       num_sms=NUM_SMS, save_for_backward=True).info()["plan"]
        seen.append(re.search(r" (LOCAL|GLOBAL|STREAM)\(", plan).group(1))
    assert len(seen) >= 6 and plans <= set(seen), seen
