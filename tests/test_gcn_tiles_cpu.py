"""CPU: the batches and plans of tests/test_gpu_gcn_tiles.py, which run the fused GCN kernel on full 128-row LOCAL tiles.

``gcn_wgmma_kernel<LOCAL=true, NH>`` keeps a tile's node states in shared memory (``sH``) between layers: the gather reads row
``s - row0`` of it, the epilogue writes rows ``r`` back, and rows 64-127 belong to the second pair of warpgroups (``mh = 1``).  The
planner shrinks the row budget of a batch that cannot fill the chip (``pack_to_fill_chip``, down to 32 rows), so small test batches run
tiles of 32-40 rows and never reach rows 64-127 of a LOCAL tile.  The batches here do, at 132 SMs (an H100 SXM):

* ``span{S}``, S in 33, 64, 65, 100, 127, 128: one component of S nodes between 40 components of 3-29 nodes, so the budget cannot shrink
  below S.  In that component row 0 and row S-1 read every other node (the gather reads ``sH`` at both ends of the tile), one row's only
  entry is a self-loop, three rows have no entries (their state is the bias alone) between rows that have some, one row's only entries
  are one (i, j) pair listed twice with weights w and -w (exactly 0 in float64, rounding noise under FMA), and one entry has weight 0;
* ``span129``: the same at 129 nodes, one more than a tile: the GLOBAL plan with fixed 128-row tiles;
* ``bench``: 5 500 synthetic molecules (99 046 nodes), the ``gcn_default_batch_100k_nodes`` workload of tools/gcn_bench.py: 832 tiles
  of up to 128 rows;
* ``mol1200``: 1 200 molecules (21 707 nodes): still more tiles than SMs at a 128-row budget (on 132 and on 114 SMs), a smaller batch
  for most GPU cases.

Tests: the batches have the shapes they claim; through the host-only prepare call at 132 SMs, with bf16x3, bf16 and fp32 and with
save_for_backward on and off, every batch reaches its plan, its largest tile lies in its band, and on LOCAL plans both ends of every list
entry fall in one tile (the kernel indexes ``sH`` by ``s - row0``).  A planner change that shrinks these batches back to small tiles
fails here.
"""
import functools
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from tests import gcn_oracle as G

NUM_SMS = 132
TILE_ROWS = 128
SPANS = (33, 64, 65, 100, 127, 128)
BATCHES = ["span%d" % S for S in SPANS] + ["span129", "mol1200", "bench"]
LOCAL_BATCHES = [b for b in BATCHES if b != "span129"]
MOLECULES = {"mol1200": 1200, "bench": 5500}
BENCH_NODES, BENCH_TILES, MOL1200_NODES = 99046, 832, 21707
HIDDEN = 100


# ---------------------------------------------------------------------------------------------------------------- span batches
def span_rows(S):
    """Local row ids of the S-node component's special rows."""
    return {"head": 0, "tail": S - 1, "self_only": 1, "empty": (3, S // 2, S - 3), "cancel": 5, "cancel_src": 7, "zero": 6, "zero_src": 8}


def span_component(S, rng):
    """The entries of one connected S-node component (local ids, row i = output, column j = input) and their weights."""
    r = span_rows(S)
    others = np.arange(1, S)
    lst = [np.stack([np.zeros(S - 1, np.int64), others], 1),                                # row 0 reads every other node
           np.stack([np.full(S - 1, S - 1, np.int64), np.arange(S - 1)], 1),               # row S-1 reads every other node
           np.array([[r["self_only"], r["self_only"]]]),
           np.array([[r["cancel"], r["cancel_src"]], [r["cancel"], r["cancel_src"]]]),
           np.array([[r["zero"], r["zero_src"]]])]
    # the two hub rows sum S-1 inputs each: scaled so that their states stay of the size of the others' (the error bars are relative to
    # the largest state, and rows 64-127 must not drown in them)
    hub = 2.0 / np.sqrt(S - 1)
    w = [rng.uniform(-hub, hub, S - 1), rng.uniform(-hub, hub, S - 1), rng.uniform(-1, 1, 1)]
    cw = np.float32(rng.uniform(0.5, 1.0))
    w += [np.array([cw, -cw]), np.array([0.0])]
    special = {r["head"], r["tail"], r["self_only"], r["cancel"], *r["empty"]}
    for i in range(S):                    # every other row: a self-loop and three random inputs inside the component (the zero row too)
        if i in special:
            continue
        lst.append(np.stack([np.full(4, i, np.int64), np.concatenate([[i], rng.integers(0, S, 3)])], 1))
        w.append(rng.uniform(-1, 1, 4))
    return np.concatenate(lst).astype(np.int64), np.concatenate(w).astype(np.float32)


@functools.lru_cache(maxsize=None)
def span_batch(S, seed=0):
    """(V, shuffled [nnz, 2] list, [nnz] weights, first node of the S-node component): 20 components of 3-29 nodes, the S-node
    component, 20 more."""
    rng = np.random.default_rng(100 + S + seed)
    sizes = list(rng.integers(3, 30, 40))
    Va, la, wa = G.component_list(sizes[:20], rng)
    ls, ws = span_component(S, rng)
    Vb, lb, wb = G.component_list(sizes[20:], rng)
    lst = np.concatenate([la, ls + Va, lb + Va + S])
    w = np.concatenate([wa, ws, wb]).astype(np.float32)
    perm = rng.permutation(w.shape[0])
    return Va + S + Vb, lst[perm], w[perm], Va


# ---------------------------------------------------------------------------------------------------------------- molecule batches
@functools.lru_cache(maxsize=None)
def molecule_feed(name):
    """``packing.pack_gcn_batch`` of synthetic molecules (seed 0) at hidden 100: the plug-in's feed of one batch."""
    return packing.pack_gcn_batch(packing.process_raw_graphs_gcn(synthetic.make_molecules(MOLECULES[name], seed=0)), HIDDEN)


def batch(name):
    """(V, [nnz, 2] list, [nnz] float32 weights) of a batch kind."""
    if name.startswith("span"):
        V, lst, w, _ = span_batch(int(name[4:]))
        return V, lst, w
    f = molecule_feed(name)
    return f["initial_node_representation"].shape[0], f["adjacency_list"], f["adjacency_weights"].astype(np.float32)


def band(name):
    """(least, most) rows of the largest tile a wgmma plan of the batch runs."""
    if name == "span129":
        return TILE_ROWS, TILE_ROWS                 # GLOBAL: fixed 128-row tiles
    if name.startswith("span"):
        return int(name[4:]), TILE_ROWS
    return TILE_ROWS, TILE_ROWS


def plan_pattern(name, precision):
    if precision == "fp32":
        return r"^gcn-fp32-ffma GLOBAL\("
    return r"^gcn-wgmma-%s %s\(" % (precision, "GLOBAL" if name == "span129" else "LOCAL")


def tile_of(tile_start, nodes):
    return np.searchsorted(tile_start, nodes, side="right") - 1


def check_tiles(name, tile_start, lst, local):
    """The largest tile lies in the batch's band; on a LOCAL plan both ends of every entry lie in one tile (and ``bench`` has its 832
    tiles).  Returns the largest tile."""
    ts = np.asarray(tile_start)
    largest = int(np.max(np.diff(ts)))
    lo, hi = band(name)
    assert lo <= largest <= hi, (name, largest, (lo, hi))
    if local:
        np.testing.assert_array_equal(tile_of(ts, lst[:, 0]), tile_of(ts, lst[:, 1]), err_msg=name)
        if name == "bench":
            assert ts.shape[0] - 1 == BENCH_TILES, ts.shape[0] - 1
    return largest


def host_graph(name, precision, save, num_sms=NUM_SMS, D=HIDDEN):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    V, lst, w = batch(name)
    return PreparedGraph.host_only_gcn(D, 3, V, lst, w, use_bias=True, precision=precision, num_sms=num_sms, save_for_backward=save)


def _clean_env(monkeypatch):
    monkeypatch.delenv("GGNN_FORCE_GLOBAL", raising=False)


# ---------------------------------------------------------------------------------------------------------------- tests
def _components(V, lst):
    """Component id of every node (union-find over the list's pairs)."""
    parent = np.arange(V)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for i, j in lst:
        a, b = find(int(i)), find(int(j))
        if a != b:
            parent[max(a, b)] = min(a, b)
    return np.array([find(x) for x in range(V)])


@pytest.mark.parametrize("S", SPANS + (129,))
def test_span_batches_have_the_shapes_they_claim(S):
    V, lst, w, off = span_batch(S)
    r = {k: (tuple(off + x for x in v) if isinstance(v, tuple) else off + v) for k, v in span_rows(S).items()}
    comp = _components(V, lst)
    members = np.flatnonzero(comp == comp[off])
    np.testing.assert_array_equal(members, np.arange(off, off + S))              # one component of exactly S nodes
    sizes = np.bincount(comp)
    assert np.sort(sizes[sizes > 0])[-2] <= 29                                     # every other component is small
    rows = lambda i: lst[lst[:, 0] == i]
    weights = lambda i: w[lst[:, 0] == i]
    span = set(range(off, off + S))
    assert set(rows(r["head"])[:, 1].tolist()) == span - {r["head"]}
    assert set(rows(r["tail"])[:, 1].tolist()) == span - {r["tail"]}
    assert rows(r["self_only"]).tolist() == [[r["self_only"], r["self_only"]]]
    for e in r["empty"]:
        assert rows(e).shape[0] == 0 and rows(e - 1).shape[0] > 0 and rows(e + 1).shape[0] > 0, e
    assert rows(r["cancel"]).tolist() == [[r["cancel"], r["cancel_src"]]] * 2
    cw = weights(r["cancel"])
    assert cw[0] == -cw[1] != 0
    assert np.any((lst[:, 0] == r["zero"]) & (lst[:, 1] == r["zero_src"]) & (w == 0.0))
    # float64: the +-w row of S is exactly 0 and its output is the bias alone; an empty row's too
    rng = np.random.default_rng(S)
    h0 = rng.normal(0, 1, (V, 8))
    k, b = G.glorot((8, 8), rng), rng.normal(0, 0.2, 8).astype(np.float32)
    out = G.gcn_propagation_loops(h0, lst, w, [k], [b])
    for i in (r["cancel"],) + r["empty"]:
        np.testing.assert_array_equal(out[i], b.astype(np.float64))


def test_molecule_batches_have_the_shapes_they_claim():
    for name, V in (("bench", BENCH_NODES), ("mol1200", MOL1200_NODES)):
        f = molecule_feed(name)
        v, lst, w = batch(name)
        assert v == V and f["num_graphs"] == MOLECULES[name], (name, v)
        assert lst.min() >= 0 and lst.max() < V and w.dtype == np.float32
        comp = np.bincount(_components(V, lst))
        assert comp.max() <= TILE_ROWS, (name, comp.max())


@pytest.mark.parametrize("save", [False, True], ids=["nosave", "save"])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "fp32"])
@pytest.mark.parametrize("name", BATCHES)
def test_batch_reaches_its_plan_and_tiles(name, precision, save, monkeypatch):
    _clean_env(monkeypatch)
    g = host_graph(name, precision, save)
    plan = g.info()["plan"]
    assert re.search(plan_pattern(name, precision), plan), (name, precision, plan)
    if precision != "fp32":
        _, lst, _ = batch(name)
        check_tiles(name, g.arrays(1)["tile_start"], lst, "LOCAL" in plan)


@pytest.mark.parametrize("D", [12, 64, 128])
def test_tiles_do_not_depend_on_the_hidden_size(D, monkeypatch):
    """The GPU file runs hidden 12..128 (NH 8..64): the same tiles at every one."""
    _clean_env(monkeypatch)
    for name in LOCAL_BATCHES:
        a = host_graph(name, "bf16x3", True, D=D).arrays(1)["tile_start"]
        np.testing.assert_array_equal(a, host_graph(name, "bf16x3", True).arrays(1)["tile_start"], err_msg=name)


def test_molecule_batches_keep_128_row_tiles_on_114_sms(monkeypatch):
    """An H100 PCIe has 114 SMs: the molecule batches still have more 128-row tiles than that, so their budget stays 128."""
    _clean_env(monkeypatch)
    for name in ("mol1200", "bench"):
        g = host_graph(name, "bf16x3", True, num_sms=114)
        assert "rows/tile<=128 " in g.info()["plan"], g.info()["plan"]
        _, lst, _ = batch(name)
        check_tiles(name, g.arrays(1)["tile_start"], lst, True)


def test_forced_global_runs_fixed_128_row_tiles(monkeypatch):
    """The LOCAL = GLOBAL comparison of the GPU file runs these batches again under GGNN_FORCE_GLOBAL=1."""
    _clean_env(monkeypatch)
    monkeypatch.setenv("GGNN_FORCE_GLOBAL", "1")
    for name in LOCAL_BATCHES:
        g = host_graph(name, "bf16x3", True)
        assert g.info()["plan"].startswith("gcn-wgmma-bf16x3 GLOBAL("), g.info()["plan"]
        V = g.info()["num_nodes"]
        np.testing.assert_array_equal(g.arrays(1)["tile_start"], list(range(0, V, TILE_ROWS)) + [V])
