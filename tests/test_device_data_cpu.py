"""CPU: the host half of a device-resident dataset batch (``ggnn_dataset_prepare_batch``) against the edge-list builder.

A dataset batch is planned from per-graph summaries only (node and message counts, cut segments); the packers' path builds the same batch
from its concatenated edge lists (``ggnn_host_prepare_graph_sparse`` / ``_gcn``).  Both must give the same plan -- plan text, tile starts,
node and message counts, streaming or not, image size -- for every batch, model shape and SM count.  The image bytes themselves are
compared on the GPU (tests/test_gpu_device_data.py)."""
import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GgnnError, PreparedGraph

GRU = {"layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "use_edge_bias": False, "use_edge_msg_avg_aggregation": True,
       "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}
T = 4
ANN = 5


def _graph(n, edges_per_type, seed, label=0.5):
    """A processed sparse graph (process_raw_graphs_sparse's schema) with the given graph-local (source, target) lists per type."""
    rng = np.random.default_rng(seed)
    adj, indeg = {}, {}
    for e, pairs in edges_per_type.items():
        a = np.asarray(pairs, np.int32).reshape(-1, 2)
        adj[e] = a
        nodes, counts = np.unique(a[:, 1], return_counts=True)
        indeg[e] = {int(v): int(c) for v, c in zip(nodes, counts)}
    return {"adjacency_lists": adj, "num_incoming_edge_per_type": indeg, "init": rng.normal(size=(n, ANN)).astype(np.float32).tolist(),
            "labels": [label, None if seed % 3 == 0 else -label]}


def hand_made_graphs():
    """A graph larger than a 128-row tile, interleaved components, a single node, types without edges, a graph without any edge."""
    chain = [(i, i + 1) for i in range(299)]
    big = _graph(300, {0: chain + [(j + 1, j) for j, _ in chain], 2: [(0, 150), (150, 0), (10, 10)]}, 1)
    inter = _graph(12, {1: [(0, 2), (2, 4), (4, 0), (1, 3), (3, 5), (7, 11), (11, 7)], 3: [(2, 0), (2, 0), (6, 8)]}, 2)
    single = _graph(1, {}, 3)
    sparse_types = _graph(7, {3: [(0, 1), (1, 0), (5, 6), (6, 5), (6, 6)]}, 4)
    return [big, inter, single, sparse_types]


def sparse_graph_set(n_mol=60, seed=0):
    mols = synthetic.make_molecules(n_mol, seed=seed, num_bond_types=T)
    graphs = packing.process_raw_graphs_sparse(mols)
    for g in graphs:
        g["labels"] = g["labels"] + [None if len(g["init"]) % 2 else 1.25]
    return graphs + hand_made_graphs()


def gcn_graph_set(n_mol=60, seed=0):
    mols = synthetic.make_molecules(n_mol, seed=seed, num_bond_types=T)
    graphs = packing.process_raw_graphs_gcn(mols)
    for g in hand_made_graphs():
        n = len(g["init"])
        lst = np.concatenate([a for a in g["adjacency_lists"].values()] + [np.zeros((0, 2), np.int32)])[:, ::-1].astype(np.int64)
        lst = np.concatenate([lst, np.stack([np.arange(n), np.arange(n)], 1)])
        w = np.linspace(0.25, 1.0, lst.shape[0])
        graphs.append({"adjacency_list": lst, "adjacency_weights": w, "init": g["init"], "labels": [g["labels"][0]]})
    return graphs


def batch_ids(N, seed):
    """Seeded batches: random subsets in random order (repeats allowed), each hand-made graph alone and together, and the empty batch."""
    rng = np.random.default_rng(seed)
    out = [rng.integers(0, N, size=int(rng.integers(1, 40))) for _ in range(12)]
    out += [np.array([i]) for i in range(N - 4, N)] + [np.arange(N - 4, N)[::-1], np.array([N - 1, 0, N - 3, 5, N - 4]), np.zeros(0, np.int64)]
    return out


def packed_graph(flat, ids, hidden):
    """The batch through the packer (an empty batch, which the packer cannot pack, as empty lists)."""
    if len(ids) == 0:
        if isinstance(flat, packing.FlatGCNGraphs):
            return {"initial_node_representation": np.zeros((0, hidden), np.float32), "adjacency_list": np.zeros((0, 2), np.int64),
                    "adjacency_weights": np.zeros(0)}
        return {"adjacency_lists": [np.zeros((0, 2), np.int32)] * flat.num_edge_types,
                "num_incoming_edges_per_type": np.zeros((0, flat.num_edge_types), np.float32)}
    return flat.pack(ids, hidden)


def tile_starts(ref, T):
    """The reference's tile starts (an empty batch has the one entry 0; its arrays() would not size the streaming table of an empty batch)."""
    return ref.arrays(T)["tile_start"] if ref.info()["num_nodes"] else np.zeros(1, np.int32)


def plan_of(info):
    return (info["num_nodes"], info["num_messages"], info["num_tiles"], info["image_bytes"], info["streaming"], info["plan"])


SPARSE_CASES = [  # (hidden, precision, attention, num_sms)
    (100, "bf16x3", False, 132), (100, "fp32", False, 132), (256, "bf16x3", False, 132), (100, "fp32", True, 132), (100, "bf16x3", False, 16),
    (24, "bf16", False, 8),
]


@pytest.mark.parametrize("hidden,precision,att,num_sms", SPARSE_CASES)
@pytest.mark.parametrize("save", [False, True])
def test_sparse_batch_plan_equals_edge_list_builder(hidden, precision, att, num_sms, save):
    graphs = sparse_graph_set()
    flat = packing.FlatSparseGraphs(graphs, T)
    params = dict(GRU, hidden_size=hidden, use_propagation_attention=att)
    ds = DeviceDataset.host_only(params, T, flat, precision=precision, num_sms=num_sms, for_training=save)
    for ids in batch_ids(flat.num_graphs, seed=hidden + num_sms):
        b = ds.prepare_batch(ids, save_for_backward=save)
        packed = packed_graph(flat, ids, hidden)
        ref = PreparedGraph.host_only(params, T, packed["adjacency_lists"], packed["num_incoming_edges_per_type"], precision=precision,
                                      num_sms=num_sms, save_for_backward=save)
        got, want = b.info(), ref.info()
        assert plan_of(got) == plan_of(want), ids
        np.testing.assert_array_equal(got["tile_start"], tile_starts(ref, T))
        if "LOCAL" in want["plan"]:   # what the tile-local launches size their shared memory by
            assert (got["max_tile_msgs"], got["max_tile_types"]) == ref.tile_stats(), ids


@pytest.mark.parametrize("hidden,precision,num_sms", [(100, "bf16x3", 132), (100, "fp32", 132), (200, "bf16x3", 132), (64, "bf16x3", 16)])
@pytest.mark.parametrize("save", [False, True])
def test_gcn_batch_plan_equals_edge_list_builder(hidden, precision, num_sms, save):
    flat = packing.FlatGCNGraphs(gcn_graph_set())
    ds = DeviceDataset.host_only_gcn(hidden, 3, flat, precision=precision, num_sms=num_sms, for_training=save)
    for ids in batch_ids(flat.num_graphs, seed=hidden):
        b = ds.prepare_batch(ids, save_for_backward=save)
        packed = packed_graph(flat, ids, hidden)
        ref = PreparedGraph.host_only_gcn(hidden, 3, packed["initial_node_representation"].shape[0], packed["adjacency_list"],
                                          packed["adjacency_weights"], precision=precision, num_sms=num_sms, save_for_backward=save)
        got, want = b.info(), ref.info()
        assert plan_of(got) == plan_of(want), ids
        np.testing.assert_array_equal(got["tile_start"], tile_starts(ref, 1))
        if "LOCAL" in want["plan"]:   # what the tile-local launches size their shared memory by
            assert (got["max_tile_msgs"], got["max_tile_types"]) == ref.tile_stats(), ids


def test_a_batch_rebuilt_in_place_plans_like_a_fresh_one():
    flat = packing.FlatSparseGraphs(sparse_graph_set(), T)
    params = dict(GRU, hidden_size=100)
    ds = DeviceDataset.host_only(params, T, flat, precision="bf16x3")
    b = ds.prepare_batch(np.arange(flat.num_graphs))
    small = np.array([3, 1])
    assert plan_of(ds.prepare_batch(small, reuse=b).info()) == plan_of(ds.prepare_batch(small).info())


def test_refusals_carry_the_documented_codes():
    graphs = sparse_graph_set(8)
    flat = packing.FlatSparseGraphs(graphs, T)
    params = dict(GRU, hidden_size=100)
    ds = DeviceDataset.host_only(params, T, flat, precision="bf16x3", for_training=False)
    for bad in ([0, flat.num_graphs], [-1]):
        with pytest.raises(GgnnError, match="out of range") as ex:
            ds.prepare_batch(bad, save_for_backward=False)
        assert ex.value.code == -5   # GGNN_ERANGE
    with pytest.raises(GgnnError, match="created for training") as ex:   # no source-keyed CSR in this dataset
        ds.prepare_batch([0], save_for_backward=True)
    assert ex.value.code == -3       # GGNN_ESTATE

    broken = [dict(g) for g in graphs]
    n = len(broken[2]["init"])
    broken[2]["adjacency_lists"] = {**broken[2]["adjacency_lists"], 1: np.array([[0, n]], np.int32)}   # target outside graph 2
    with pytest.raises(GgnnError, match="graph 2: edge 0 of type 1") as ex:
        DeviceDataset.host_only(params, T, packing.FlatSparseGraphs(broken, T), precision="bf16x3")
    assert ex.value.code == -5

    gflat = packing.FlatGCNGraphs(gcn_graph_set(4))
    gflat.lists = gflat.lists.copy()
    gflat.lists[gflat.entry_off[1]] = (0, int(gflat.n_nodes[1]))   # first entry of graph 1, column outside it
    with pytest.raises(GgnnError, match="graph 1: entry 0") as ex:
        DeviceDataset.host_only_gcn(64, 2, gflat)
    assert ex.value.code == -5


def test_device_data_option_is_not_a_param_and_needs_a_gpu(tmp_path):
    """--device-data is a command-line option: params (what a checkpoint must match) do not change, and a CPU device is refused."""
    from gated_graph_neural_network_samples_b200 import chem_gcn, chem_sparse
    mols = synthetic.make_molecules(8, seed=1)
    args = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:6], "--valid_data": mols[6:], "--config": {"hidden_size": 16}}
    for model in (chem_sparse.SparseGGNNChemModel, chem_gcn.SparseGCNChemModel):
        assert model._resolve_params(dict(args, **{"--device-data": True})) == model._resolve_params(args)
        with pytest.raises(Exception, match="--device-data .* needs a CUDA device"):
            model(dict(args, **{"--device-data": True}))
