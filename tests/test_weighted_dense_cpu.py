"""CPU: the weighted dense batches of tests/test_gpu_weighted_dense.py, their shapes, the float64 oracle on them, and the plans of their
binary twins.

A weighted ``[b, T, v, v]`` matrix fed through ``ggnn_set_graph_dense`` is scanned (``scan_dense``) into per-type message lists, per-slot
weights and fp32 row sums, and every forward and backward kernel then scales each message by its slot weight.  The GPU file holds each of
those kernels to the float64 dense oracle; this file makes sure that what it feeds them is what it claims:

* every batch has the shape its cases rely on (component sizes, node count, edge types present), and every weight regime the values it
  names (negative entries, rows whose fp32 sum is exactly 0, exact 1.0 entries, per-graph scales, a single non-0/1 entry in the last
  graph);
* the two dense oracle statements (``dense_propagation_loops``, ``dense_propagation_torch``) agree in float64 to 1e-12 on every batch and
  regime, with and without edge bias, so that a difference on the GPU is the kernel's;
* the host-only dense prepare refuses weighted matrices, so the weighted plan text is asserted on the device.  What can be pinned here
  is the binary twin (the same nonzero pattern with every entry 1): it has the same components, so the same tiles, and at 132 SMs (an
  H100 SXM) under the case's environment its plan must be the family the weighted case claims.  The one exception is the tensor-core
  batch with a 200-node component: unweighted it streams, weighted it must stay on the tile kernel's GLOBAL plan;
* the binary prepare refuses every weighted regime at every host thread count, the matrix whose only non-0/1 entry lies in its last
  graph included: the scan must see that entry whichever thread's range it falls in.
"""
import functools
import os
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from oracle import ggnn_oracle as O
from tests import _util as U
from tests.test_backward_plans_cpu import FORCE_GLOBAL, plan_matches
from tests.test_forward_plans_cpu import BIG_SIZES, pad16

NUM_SMS = 132
WEIGHTED_TAG = " [weighted dense adjacency -> weighted CSR]"
BINARY_TAG = " [binary dense adjacency -> CSR]"
HOST_THREADS = (1, 2, 3, 8)


# ---------------------------------------------------------------------------------------------------------------- binary patterns
def _connect(A, g, n, rng, types, extra):
    """Graph ``g`` of ``A``: one connected component on nodes 0..n-1 (a random spanning tree plus ``extra`` distinct extra pairs), both
    directions, each undirected edge of a type drawn from ``types`` (the first ones in order, so that every listed type occurs)."""
    pairs = [(int(rng.integers(0, i)), i) for i in range(1, n)]
    seen = set(pairs)
    extra = min(extra, n * (n - 1) // 2 - len(pairs))
    while extra > 0:
        a, c = sorted(int(x) for x in rng.choice(n, 2, replace=False))
        if (a, c) not in seen:
            seen.add((a, c))
            pairs.append((a, c))
            extra -= 1
    for k, (a, c) in enumerate(pairs):
        t = types[k] if k < len(types) else types[int(rng.integers(0, len(types)))]
        A[g, t, c, a] = A[g, t, a, c] = 1.0


def components(sizes, v, T, seed, types=None, extra_per_node=1.0):
    """``[b, T, v, v]`` 0/1 matrix: graph g one component of ``sizes[g]`` nodes, its other v - sizes[g] nodes isolated."""
    rng = np.random.default_rng(seed)
    A = np.zeros((len(sizes), T, v, v), np.float32)
    for g, n in enumerate(sizes):
        _connect(A, g, n, rng, list(types if types is not None else range(T)), int(extra_per_node * n))
    return A


def molecules(n, v=29, T=4, seed=8):
    mols = synthetic.make_molecules(n, seed=seed, num_bond_types=T)
    return np.asarray(packing.pack_dense_batch(mols, v, 8, T)["adjacency_matrix"], np.float32)   # (the 5 node features need hidden >= 5)


def tail_columns(v, b=12, T=4, seed=0):
    """Entries only in the columns the scan visits one float at a time (j >= v - v % 4): for v = 1, 2, 3 every column, for v = 5 only
    column 4, so every message of the batch has source node 4 of its graph (node 4's own row included: a self-loop)."""
    rng = np.random.default_rng(seed + v)
    A = np.zeros((b, T, v, v), np.float32)
    tail = list(range(v - v % 4, v))
    for g in range(b):
        for _ in range(2 * v):
            A[g, int(rng.integers(0, T)), int(rng.integers(0, v)), tail[int(rng.integers(0, len(tail)))]] = 1.0
    A[0, 0, v - 1, tail[0]] = 1.0          # (at least one entry per batch)
    return A


def with_self_loops(A, seed=3):
    """Every third node of every graph gets a self-loop of a random type, padded (isolated) nodes included: some nodes then receive
    only their own state."""
    A = A.copy()
    rng = np.random.default_rng(seed)
    b, T, v, _ = A.shape
    for g in range(b):
        for i in range(0, v, 3):
            A[g, int(rng.integers(0, T)), i, i] = 1.0
    return A


@functools.lru_cache(maxsize=None)
def _binary(name):
    if name == "mol":            # 10 molecules of at most 29 atoms: compact LOCAL tiles, both fp32 variants LOCAL
        return molecules(10)
    if name == "mol64":          # 64 molecules: the scan splits them over host threads
        return molecules(64, seed=9)
    if name == "b1":
        return molecules(1, seed=10)
    if name == "big":            # components of 66-120 nodes: 128-row LOCAL tiles
        return components(BIG_SIZES, 120, 4, 40, extra_per_node=1.0)
    if name == "one200":         # two graphs of one 200-node component each: GLOBAL
        return components((200, 200), 200, 4, 41, extra_per_node=1.0)
    if name == "T1":
        return components(list(np.random.default_rng(42).integers(3, 20, 12)), 20, 1, 42)
    if name == "T16":            # 16 types, only 0, 7 and 15 present
        return components(list(np.random.default_rng(43).integers(3, 20, 12)), 20, 16, 43, types=(0, 7, 15))
    if name == "selfloop":
        return with_self_loops(molecules(10))
    m = re.match(r"^v(\d+)$", name)
    if m:
        return tail_columns(int(m.group(1)))
    raise ValueError(name)


def binary(name):
    return _binary(name).copy()


# ---------------------------------------------------------------------------------------------------------------- weight regimes
REGIMES = ("binary", "uniform", "signed", "ones", "scales", "lastonly")


def weigh(Abin, regime, seed=2):
    """The regime's weights on the nonzero pattern of ``Abin``:

    * ``uniform``: U(0.25, 1.75);
    * ``signed``: k / 64 with |k| in [16, 112] and random sign; in every other row (graph, type, target) of two or more entries the first
      ones positive and the last minus their sum, so that the row's fp32 sum is exactly 0 (the values are dyadic: every partial sum is
      exact) and its edge-bias term vanishes;
    * ``ones``: uniform with about a third of the entries exactly 1.0;
    * ``scales``: uniform times a per-graph scale from 1e-3 to 1e3 (log-spaced over the graphs);
    * ``lastonly``: 0/1 except one entry of the last graph, 0.5;
    * ``binary``: the 0/1 pattern itself."""
    rng = np.random.default_rng(seed)
    nz = Abin != 0
    if regime == "binary":
        return nz.astype(np.float32)
    if regime in ("uniform", "ones", "scales"):
        A = np.where(nz, rng.uniform(0.25, 1.75, Abin.shape), 0.0).astype(np.float32)
        if regime == "ones":
            A[nz & (rng.random(Abin.shape) < 1 / 3)] = 1.0
        if regime == "scales":
            A *= np.logspace(-3, 3, Abin.shape[0]).astype(np.float32)[:, None, None, None]
        return A
    if regime == "signed":
        k = rng.integers(16, 113, Abin.shape) * rng.choice((-1, 1), Abin.shape)
        A = np.where(nz, k / 64.0, 0.0).astype(np.float32)
        rows = np.argwhere(nz.sum(-1) >= 2)
        for g, t, i in rows[::2]:
            cols = np.flatnonzero(nz[g, t, i])
            vals = rng.integers(16, 113, len(cols) - 1) / 64.0
            A[g, t, i, cols[:-1]] = vals
            A[g, t, i, cols[-1]] = -vals.sum()
        return A
    if regime == "lastonly":
        A = nz.astype(np.float32)
        g, t, i, j = np.argwhere(nz[-1:])[0]
        A[Abin.shape[0] - 1, t, i, j] = 0.5
        return A
    raise ValueError(regime)


def h0_for(A, D, seed=0):
    b, _, v, _ = A.shape
    return np.random.default_rng(500 + D + seed).normal(0, 1, (b, v, D)).astype(np.float32)


def case_h0(c, A):
    """h0 of a case.  The ``scales`` regime divides the states of each graph whose weights are scaled up by its scale, so that its messages
    stay O(1): with O(1) states, weights of 10 and more make the propagation itself ill-conditioned (the float32 restatement of the oracle
    is 4e-3 off float64 on such a graph after three steps), which no fp32 kernel can meet at 1e-5."""
    h0 = h0_for(A, c.D)
    if c.regime == "scales":
        h0 = (h0 / np.maximum(np.logspace(-3, 3, A.shape[0]), 1.0)[:, None, None]).astype(np.float32)
    return h0


# ---------------------------------------------------------------------------------------------------------------- the GPU file's cases
def tc_pattern(prec, kind, DP):
    """Plan text of the tile-local wgmma kernel: compact 64-row LOCAL tiles, 128-row LOCAL tiles (a row budget of 65-128 rows, no
    compact operand tiles), or GLOBAL."""
    if kind == "compact":
        return r"^wgmma-%s LOCAL\(.* \(compact 64-row operand tiles\) DP=%d " % (prec, DP)
    if kind == "128":
        return r"^wgmma-%s LOCAL\(.* rows/tile<=(?:6[5-9]|[7-9]\d|1[01]\d|12[0-8]) DP=%d " % (prec, DP)
    return r"^wgmma-%s GLOBAL\(.* DP=%d " % (prec, DP)


def ffma_pattern(variant, nb1, local):
    rows, cs = (64, 1) if variant == 0 else (32, 2)
    return r"^fp32-ffma %s\(.* rows/tile<=%d warps=8 colsplit=%d nb1=%d " % ("LOCAL" if local else "GLOBAL", rows, cs, nb1)


STEPWISE = r"^fp32-stepwise \("


class Case:
    """One weighted dense forward: batch, weight regime, precision, hidden size, environment, plan-text pattern (without the weighted
    suffix), and the model: ``steps`` timesteps, edge bias on / off, state keep probability.  ``twin``: the pattern the binary twin's
    host-only plan must match (None: pin the case's own pattern)."""

    def __init__(self, name, batch, regime, precision, D, env, pattern, steps=3, bias=True, keep=1.0, twin=None):
        self.name, self.batch, self.regime, self.precision, self.D = name, batch, regime, precision, D
        self.env, self.pattern, self.steps, self.bias, self.keep, self.twin = dict(env), pattern, steps, bias, keep, twin

    @property
    def params(self):
        return U.dense_params_as_engine_params({"num_timesteps": self.steps, "use_edge_bias": self.bias}, self.D)

    def matrix(self):
        return weigh(binary(self.batch), self.regime)

    def __repr__(self):
        return self.name


def _tile_cases():
    """1. The tile-local wgmma kernel at every NH, D = 2 NH and 2 NH - 4 in turn, bf16x3 and bf16: compact LOCAL, 128-row LOCAL, GLOBAL
    through a 200-node component (no environment variable), and forced GLOBAL on molecules."""
    out = []
    for nh in range(8, 65, 8):
        DP = 2 * nh
        Ds = (DP, max(DP - 4, 4))
        for i, prec in enumerate(("bf16x3", "bf16")):
            Da, Db = Ds[i], Ds[1 - i]
            stream = r"^wgmma-%s STREAM\(" % prec
            out += [Case("tc-nh%d-%s-compact-D%d" % (nh, prec, Da), "mol", "uniform", prec, Da, {}, tc_pattern(prec, "compact", DP)),
                    Case("tc-nh%d-%s-local128-D%d" % (nh, prec, Db), "big", "uniform", prec, Db, {}, tc_pattern(prec, "128", DP)),
                    Case("tc-nh%d-%s-global-D%d" % (nh, prec, Da), "one200", "uniform", prec, Da, {}, tc_pattern(prec, "global", DP),
                         twin=stream),
                    Case("tc-nh%d-%s-forced-global-D%d" % (nh, prec, Db), "mol", "uniform", prec, Db, FORCE_GLOBAL,
                         tc_pattern(prec, "global", DP))]
    return out


def _ffma_cases():
    """2. All twelve fp32 instances at the hidden sizes tests/test_forward_plans_cpu.py uses for them."""
    out = []
    for v, sizes in enumerate(((28, 60, 100), (44, 116, 196))):
        for nb1, D in zip((1, 2, 4), sizes):
            for loc in (True, False):
                env = {"GGNN_FFMA_VARIANT": str(v)}
                env.update({} if loc else FORCE_GLOBAL)
                out.append(Case("ffma-v%d-nb%d-%s-D%d" % (v, nb1, "local" if loc else "global", D), "mol", "uniform", "fp32", D, env,
                                ffma_pattern(v, nb1, loc)))
    return out


def _stepwise_cases():
    """3. The per-timestep fp32 path above hidden 256."""
    return [Case("stepwise-D%d" % D, "mol", "uniform", "fp32", D, {}, STEPWISE) for D in (260, 512)]


# edge kinds: (batch, regime, model overrides)
EDGE_KINDS = {
    "T1": ("T1", "uniform", {}),
    "T16-few": ("T16", "uniform", {}),
    "no-bias": ("mol", "uniform", {"bias": False}),
    "steps1": ("mol", "uniform", {"steps": 1}),
    "steps8": ("mol", "uniform", {"steps": 8}),
    "keep08": ("mol", "uniform", {"keep": 0.8}),
    "b1": ("b1", "uniform", {}),
    "v1": ("v1", "uniform", {}),
    "v2": ("v2", "uniform", {}),
    "v3": ("v3", "uniform", {}),
    "v5": ("v5", "uniform", {}),
    "self-loops": ("selfloop", "uniform", {}),
    "signed": ("mol", "signed", {}),
    "ones": ("mol", "ones", {}),
    "scales": ("mol", "scales", {"steps": 1, "bias": False}),   # (one step on O(1) messages: see case_h0)
    "last-only": ("mol64", "lastonly", {}),
}


def _edge_cases():
    """4. The edge kinds at hidden 36 and 100, fp32 and bf16x3, LOCAL and GLOBAL."""
    out = []
    for kind, (batch, regime, kw) in EDGE_KINDS.items():
        for D in (36, 100):
            for prec in ("fp32", "bf16x3"):
                for loc in (True, False):
                    if prec == "fp32":
                        pat = r"^fp32-ffma %s\(" % ("LOCAL" if loc else "GLOBAL")
                    else:
                        pat = r"^wgmma-bf16x3 %s\(.* DP=%d " % ("LOCAL" if loc else "GLOBAL", pad16(D))
                    out.append(Case("edge-%s-%s-%s-D%d" % (kind, prec, "local" if loc else "global", D), batch, regime, prec, D,
                                    {} if loc else FORCE_GLOBAL, pat, **kw))
    return out


TILE, FFMA, STEP, EDGE = _tile_cases(), _ffma_cases(), _stepwise_cases(), _edge_cases()
CASES = {c.name: c for c in TILE + FFMA + STEP + EDGE}
assert len(CASES) == len(TILE + FFMA + STEP + EDGE), "duplicate case names"

# gradients: one case per plan family (tc compact / 128-row / GLOBAL with a bf16x3 forward, fp32 variant 0 and 1 LOCAL, fp32 GLOBAL,
# stepwise), and the signed / cancelling regime on one LOCAL and one GLOBAL case.  Every one with state dropout 0.8.
GRAD = [Case("grad-tc-compact-D100", "mol", "uniform", "bf16x3", 100, {}, tc_pattern("bf16x3", "compact", 112), keep=0.8),
        Case("grad-tc-local128-D100", "big", "uniform", "bf16x3", 100, {}, tc_pattern("bf16x3", "128", 112), keep=0.8),
        Case("grad-tc-global-D100", "one200", "uniform", "bf16x3", 100, {}, tc_pattern("bf16x3", "global", 112), keep=0.8,
             twin=r"^wgmma-bf16x3 STREAM\("),
        Case("grad-ffma0-local-D100", "mol", "uniform", "fp32", 100, {"GGNN_FFMA_VARIANT": "0"}, ffma_pattern(0, 4, True), keep=0.8),
        Case("grad-ffma1-local-D36", "mol", "uniform", "fp32", 36, {"GGNN_FFMA_VARIANT": "1"}, ffma_pattern(1, 1, True), keep=0.8),
        Case("grad-ffma-global-D100", "mol", "uniform", "fp32", 100, dict(FORCE_GLOBAL, GGNN_FFMA_VARIANT="0"), ffma_pattern(0, 4, False),
             keep=0.8),
        Case("grad-stepwise-D260", "mol", "uniform", "fp32", 260, {}, STEPWISE, keep=0.8),
        Case("grad-ffma1-local-signed-D36", "mol", "signed", "fp32", 36, {"GGNN_FFMA_VARIANT": "1"}, ffma_pattern(1, 1, True), keep=0.8),
        Case("grad-tc-global-signed-D100", "one200", "signed", "bf16x3", 100, {}, tc_pattern("bf16x3", "global", 112), keep=0.8,
             twin=r"^wgmma-bf16x3 STREAM\(")]
GRAD_CASES = {c.name: c for c in GRAD}
DETERMINISM = ["grad-tc-local128-D100", "grad-tc-global-D100", "grad-ffma-global-D100", "grad-tc-global-signed-D100"]
ALL_CASES = dict(CASES, **GRAD_CASES)


def host_plan_of_twin(c):
    """The host-only plan text of case ``c``'s binary twin at 132 SMs, under the case's environment."""
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    saved = {k: os.environ.get(k) for k in c.env}
    os.environ.update(c.env)
    try:
        twin = weigh(binary(c.batch), "binary")
        return PreparedGraph.host_only_dense(c.params, twin.shape[1], twin, precision=c.precision, num_sms=NUM_SMS).info()["plan"]
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---------------------------------------------------------------------------------------------------------------- tests
def _component_sizes(Ag):
    """Connected component sizes of one graph's [T, v, v] matrix (any type, either direction)."""
    from scipy.sparse.csgraph import connected_components
    m = (Ag != 0).any(0)
    _, lab = connected_components(m | m.T, directed=False)
    return np.bincount(lab)


def test_batches_have_the_shapes_the_cases_claim():
    """Component sizes, node counts and edge types present."""
    mol = binary("mol")
    assert mol.shape == (10, 4, 29, 29) and all(_component_sizes(g).max() <= 29 for g in mol)
    assert all(mol[:, t].any() for t in range(4))
    assert binary("mol64").shape[0] == 64 and binary("b1").shape[0] == 1
    big = binary("big")
    assert big.shape == (5, 4, 120, 120)
    assert sorted(_component_sizes(g).max() for g in big) == sorted(BIG_SIZES) and 64 < min(BIG_SIZES) and max(BIG_SIZES) <= 128
    one = binary("one200")
    assert one.shape == (2, 4, 200, 200) and all(list(_component_sizes(g)) == [200] for g in one)    # one component > 128 nodes
    assert binary("T1").shape[1] == 1
    t16 = binary("T16")
    assert t16.shape[1] == 16 and [t for t in range(16) if t16[:, t].any()] == [0, 7, 15]
    for v in (1, 2, 3, 5):
        a = binary("v%d" % v)
        assert a.shape[2:] == (v, v) and a.any()
        assert not a[..., :v - v % 4].any()                      # only the scan's tail columns
    assert binary("v5")[..., 4].sum() > 10
    sl = binary("selfloop")
    diag = np.einsum("btii->bi", sl)
    assert diag.any() and (diag[:, 27:] > 0).any()                 # padded nodes with only a self-loop
    for name in ("mol", "mol64", "big", "one200", "T1", "T16", "selfloop", "v1", "v2", "v3", "v5", "b1"):
        assert set(np.unique(binary(name))) <= {0.0, 1.0}, name


@pytest.mark.parametrize("batch", ["mol", "mol64", "big", "one200", "v5"])
def test_weight_regimes_hold_what_they_name(batch):
    Abin = binary(batch)
    nz = Abin != 0
    u = weigh(Abin, "uniform")
    assert np.all((u[nz] >= 0.25) & (u[nz] <= 1.75)) and np.all(u[~nz] == 0) and np.any(u[nz] != 1.0)
    s = weigh(Abin, "signed")
    assert np.array_equal(s != 0, nz) and np.any(s < 0)
    rowsum = s.sum(-1, dtype=np.float32)
    cancel = (nz.sum(-1) >= 2) & (rowsum == 0)
    if (nz.sum(-1) >= 2).any():
        assert cancel.any()
        # exactly 0 in fp32 in the scan's column order, and in float64
        g, t, i = np.argwhere(cancel)[0]
        acc = np.float32(0)
        for x in s[g, t, i][nz[g, t, i]]:
            acc = np.float32(acc + x)
        assert acc == 0 and s[g, t, i].astype(np.float64).sum() == 0
    o = weigh(Abin, "ones")
    assert np.any(o[nz] == 1.0) and np.any(o[nz] != 1.0) and np.array_equal(o != 0, nz)
    sc = weigh(Abin, "scales")
    scale = np.logspace(-3, 3, Abin.shape[0])
    for g in range(Abin.shape[0]):
        if nz[g].any():
            assert 0.25 * scale[g] * 0.999 <= np.abs(sc[g][nz[g]]).min() and np.abs(sc[g]).max() <= 1.75 * scale[g] * 1.001
    lo = weigh(Abin, "lastonly")
    off = np.argwhere((lo != 0) & (lo != 1))
    assert len(off) == 1 and off[0][0] == Abin.shape[0] - 1 and np.array_equal(lo != 0, nz)


def _oracle_agree(A, D, bias, steps=3):
    import torch
    T = A.shape[1]
    h0 = h0_for(A, D)
    w = O.init_dense_weights({"hidden_size": D, "use_edge_bias": bias}, T, np.random.default_rng(5))
    w["cand_bias"] = np.random.default_rng(6).normal(0, 0.1, D).astype(np.float32)
    p = {"num_timesteps": steps, "use_edge_bias": bias}
    a = O.dense_propagation_loops(h0, A, w, p, dtype=np.float64)
    b = O.dense_propagation_torch(h0, A, w, p, dtype=torch.float64).numpy()
    assert U.max_rel_err(b, a) < 1e-12
    return a


ORACLE_BATCHES = ["mol", "mol64", "big", "one200", "T1", "T16", "b1", "v1", "v2", "v3", "v5", "selfloop"]


@pytest.mark.parametrize("bias", [True, False], ids=["bias", "no-bias"])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("batch", ORACLE_BATCHES)
def test_oracle_statements_agree(batch, regime, bias):
    """``dense_propagation_loops`` and ``dense_propagation_torch`` in float64, to 1e-12, on every batch and weight regime."""
    if regime == "lastonly" and binary(batch).shape[0] == 1:
        regime = "uniform"
    _oracle_agree(weigh(binary(batch), regime), 8, bias)


def test_cancelling_rows_carry_no_edge_bias():
    """In the oracle a row whose weights sum to 0 gets no edge-bias term: with zero edge weights, one step of such a row sees only the
    GRU of its own state, the same as an isolated node's."""
    Abin = binary("mol")
    s = weigh(Abin, "signed")
    D, T = 8, Abin.shape[1]
    w = O.init_dense_weights({"hidden_size": D, "use_edge_bias": True}, T, np.random.default_rng(5))
    w["edge_weights"] = np.zeros_like(w["edge_weights"])
    h0 = h0_for(s, D)
    out = O.dense_propagation_loops(h0, s, w, {"num_timesteps": 1, "use_edge_bias": True}, dtype=np.float64)
    iso = O.dense_propagation_loops(h0, np.zeros_like(s), w, {"num_timesteps": 1, "use_edge_bias": True}, dtype=np.float64)
    rows = s.sum(-1, dtype=np.float64)                              # [b, T, v]
    zero_rows = np.all(rows == 0, axis=1) & (s != 0).any(axis=(1, 3))  # every type's sum 0, at least one entry
    assert zero_rows.any()
    np.testing.assert_array_equal(out[zero_rows], iso[zero_rows])
    assert not np.allclose(out[~zero_rows & (s != 0).any(axis=(1, 3))], iso[~zero_rows & (s != 0).any(axis=(1, 3))])


@pytest.mark.parametrize("name", sorted(ALL_CASES))
def test_binary_twin_reaches_the_plan(name):
    """The binary twin of every GPU case lands, at 132 SMs, on the plan family the weighted case claims (the 200-node tensor-core
    batch: on the streaming plan, which the weighted batch may not take)."""
    c = ALL_CASES[name]
    plan = host_plan_of_twin(c)
    assert plan.endswith(BINARY_TAG), plan
    assert plan_matches(plan, c.twin or c.pattern), (c.twin or c.pattern, plan)


def test_every_kernel_instance_has_a_case():
    """Every NH of the tile kernel on each of its four weighted plans at both wgmma precisions, and all twelve fp32 instances."""
    kinds = {(c.name.split("-")[1], c.precision, c.name.split("-")[3]) for c in TILE}
    assert kinds == {("nh%d" % nh, p, k) for nh in range(8, 65, 8) for p in ("bf16x3", "bf16") for k in ("compact", "local128", "global", "forced")}
    assert {(n.split("-")[1], n.split("-")[2], n.split("-")[3]) for n in CASES if n.startswith("ffma-")} == \
        {("v%d" % v, "nb%d" % nb, loc) for v in (0, 1) for nb in (1, 2, 4) for loc in ("local", "global")}


@pytest.mark.parametrize("regime", [r for r in REGIMES if r != "binary"])
def test_binary_prepare_refuses_weighted_matrices_at_every_thread_count(regime, monkeypatch):
    """The host-only dense prepare takes 0/1 matrices only.  On 64 graphs, at 1, 2, 3 and 8 host threads, every weighted regime is
    refused, the matrix whose only non-0/1 entry is in the last graph (the last thread's range) included; its binary twin is taken, with
    the same image at every thread count."""
    from gated_graph_neural_network_samples_b200.engine import GgnnError, PreparedGraph
    Abin = binary("mol64")
    A = weigh(Abin, regime)
    p = U.dense_params_as_engine_params({"num_timesteps": 3, "use_edge_bias": True}, 36)
    images = []
    for n in HOST_THREADS:
        monkeypatch.setenv("GGNN_HOST_THREADS", str(n))
        with pytest.raises(GgnnError, match="not 0/1"):
            PreparedGraph.host_only_dense(p, 4, A, precision="bf16x3", num_sms=NUM_SMS)
        g = PreparedGraph.host_only_dense(p, 4, weigh(Abin, "binary"), precision="bf16x3", num_sms=NUM_SMS)
        assert g.info()["plan"].endswith(BINARY_TAG)
        images.append(g.image())
    for im in images[1:]:
        np.testing.assert_array_equal(im, images[0])
