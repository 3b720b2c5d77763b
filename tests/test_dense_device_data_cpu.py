"""CPU: the host half of a dense device-resident dataset batch (``ggnn_dataset_prepare_batch_dense``) against the dense builder.

The dense model's batches are bucketed: every graph of a batch gets ``v`` rows, the bucket size, and rows beyond a graph's extent are
isolated padding.  The packers' path builds the ``[b, T, v, v]`` matrix (``pack_dense_batch``) and scans it back into edge lists
(``ggnn_host_prepare_graph_dense``); a dense dataset plans the same batch from per-graph summaries.  Both must give the same plan -- plan
text, tile starts, node and message counts, streaming or not, image size, and the tile maxima of LOCAL plans -- for every bucket and
batch size, model shape, SM count, with tied and untied edge directions.  The image bytes are compared on the GPU
(tests/test_gpu_dense_device_data.py)."""
import ctypes as C

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GgnnError, PreparedGraph
from gated_graph_neural_network_samples_b200.workloads import dense_engine_params

BONDS = 4
TASKS = (0, 1)


def edge_types(tie):
    return BONDS if tie else 2 * BONDS


def params(hidden):
    return dense_engine_params({"hidden_size": hidden, "num_timesteps": 3, "use_edge_bias": True})


def _mol(graph, n_feat, seed):
    rng = np.random.default_rng(seed)
    return {"graph": graph, "node_features": rng.integers(0, 2, size=(n_feat, 5)).astype(np.float32).tolist(),
            "targets": [[float(rng.normal())], [None if seed % 2 else float(rng.normal())]]}


def hand_made_graphs():
    """(name, raw molecule, its V_g): a duplicated bond, a self-loop, an edge to a node beyond the features, no edges, a single node."""
    return [("duplicate", _mol([[0, 1, 1], [0, 1, 1], [1, 1, 0], [1, 2, 2], [2, 3, 0]], 3, 1), 3),
            ("self-loop", _mol([[1, 2, 1], [0, 1, 1], [2, 4, 2]], 4, 2), 4),
            ("beyond-features", _mol([[0, 1, 1], [1, 3, 5], [2, 2, 4]], 3, 3), 6),
            ("no-edges", _mol([], 4, 4), 4),
            ("single-node", _mol([], 1, 5), 1)]


def molecules(seed=0):
    """Synthetic molecules in every default bucket (small ones too), then the hand-made graphs."""
    mols = []
    for k, mean in enumerate((4, 8, 12, 16, 20, 25, 28)):
        mols += synthetic.make_molecules(40, seed=seed + k, mean_atoms=mean, std_atoms=2.0)
    rng = np.random.default_rng(seed)
    for m in mols:
        m["targets"] = [m["targets"][0], [None if rng.random() < 0.3 else float(rng.normal())]]
    return mols + [g for _, g, _ in hand_made_graphs()]


def dense_batches(mols, seed):
    """(graph ids, v): per default bucket b = 1, 7, 64 and 256 graphs of it (drawn with repeats), every bucket-29 graph at once, the
    hand-made graphs alone and together (one of them with V_g == v), and the empty batch."""
    rng = np.random.default_rng(seed)
    synth = len(mols) - len(hand_made_graphs())
    buckets = np.array([packing.choose_bucket(m["graph"]) for m in mols[:synth]])
    assert set(buckets.tolist()) == set(range(len(packing.DEFAULT_BUCKET_SIZES))), "a default bucket has no molecule"
    out = []
    for bk in range(len(packing.DEFAULT_BUCKET_SIZES)):
        members = np.flatnonzero(buckets == bk)
        v = int(packing.DEFAULT_BUCKET_SIZES[bk])
        out += [(rng.choice(members, size=b), v) for b in (1, 7, 64, 256)]
    out.append((np.flatnonzero(buckets == len(packing.DEFAULT_BUCKET_SIZES) - 1), 29))
    hm = [synth + i for i in range(len(hand_made_graphs()))]
    for i, (_, _, Vg) in zip(hm, hand_made_graphs()):
        out.append((np.array([i]), Vg))   # V_g == v: no padding row
        out.append((np.array([i, 3, i]), max(Vg, 4) + 3))
    out.append((np.array(hm[::-1]), 6))
    out.append((np.zeros(0, np.int64), 8))
    return out


def flat_of(mols, tie):
    return packing.FlatDenseGraphs(mols, TASKS, tie)


def packed(mols, ids, v, hidden, tie):
    """The batch through the packer (an empty batch, which the packer cannot pack, as empty arrays)."""
    if len(ids) == 0:
        return {"adjacency_matrix": np.zeros((0, edge_types(tie), v, v), np.float32), "initial_node_representation": np.zeros((0, v, hidden), np.float32),
                "node_mask": np.zeros((0, v), np.float32), "target_values": np.zeros((len(TASKS), 0), np.float32),
                "target_mask": np.zeros((len(TASKS), 0), np.float32)}
    return packing.pack_dense_batch([mols[i] for i in ids], v, hidden, edge_types(tie), TASKS, tie)


def plan_of(info):
    return (info["num_nodes"], info["num_messages"], info["num_tiles"], info["image_bytes"], info["streaming"], info["plan"])


def tile_starts(ref, T):
    return ref.arrays(T)["tile_start"] if ref.info()["num_nodes"] else np.zeros(1, np.int32)


CASES = [  # (hidden, precision, num_sms)
    (24, "bf16x3", 132), (24, "bf16", 8), (24, "fp32", 16), (100, "bf16x3", 132), (100, "bf16x3", 8), (100, "bf16", 16), (100, "fp32", 132),
    (256, "bf16x3", 132)]


@pytest.mark.parametrize("hidden,precision,num_sms", CASES)
@pytest.mark.parametrize("save", [False, True])
@pytest.mark.parametrize("tie", [True, False])
def test_dense_batch_plan_equals_dense_builder(hidden, precision, num_sms, save, tie):
    mols = molecules()
    T = edge_types(tie)
    p = params(hidden)
    ds = DeviceDataset.host_only_dense(p, T, flat_of(mols, tie), precision=precision, num_sms=num_sms, for_training=save)
    assert ds.dense
    for ids, v in dense_batches(mols, seed=hidden + num_sms):
        b = ds.prepare_batch(ids, save_for_backward=save, nodes_per_graph=v)
        ref = PreparedGraph.host_only_dense(p, T, packed(mols, ids, v, hidden, tie)["adjacency_matrix"], precision=precision,
                                            num_sms=num_sms, save_for_backward=save)
        got, want = b.info(), ref.info()
        assert plan_of(got) == plan_of(want), (ids, v)
        assert want["plan"].endswith(" [binary dense adjacency -> CSR]") and got["num_nodes"] == len(ids) * v
        np.testing.assert_array_equal(got["tile_start"], tile_starts(ref, T))
        if "LOCAL" in want["plan"]:   # what the tile-local launches size their shared memory by
            assert (got["max_tile_msgs"], got["max_tile_types"]) == ref.tile_stats(), (ids, v)


def test_dense_messages_are_the_scanned_matrix_entries():
    """Duplicates collapse, a self-loop is one entry, a node beyond the features sends and receives: the message count of each hand-made
    graph is the number of nonzero entries of its matrix."""
    mols = [g for _, g, _ in hand_made_graphs()]
    for tie in (True, False):
        ds = DeviceDataset.host_only_dense(params(24), edge_types(tie), flat_of(mols, tie), precision="bf16x3", for_training=False)
        for i, (name, _, Vg) in enumerate(hand_made_graphs()):
            nnz = int(np.count_nonzero(packed(mols, [i], Vg, 24, tie)["adjacency_matrix"]))
            assert ds.prepare_batch([i], save_for_backward=False, nodes_per_graph=Vg).info()["num_messages"] == nnz, (name, tie)


def test_flat_dense_graphs_keep_the_packer_labels():
    """Labels and masks per task as pack_dense_batch gives them (a None target -- dropped by task_sample_ratios -- has mask 0)."""
    mols = molecules()[:50]
    flat = flat_of(mols, True)
    b = packed(mols, np.arange(50), 29, 8, True)
    np.testing.assert_array_equal(flat.labels.T, b["target_values"])
    np.testing.assert_array_equal(flat.mask.T, b["target_mask"])
    assert flat.mask[:, 1].min() == 0.0 and flat.mask[:, 1].max() == 1.0
    np.testing.assert_array_equal(flat.n_nodes, [len(m["node_features"]) for m in mols])


def test_dense_refusals_carry_the_documented_codes():
    mols = molecules()
    p = params(100)
    flat = flat_of(mols, True)
    ds = DeviceDataset.host_only_dense(p, BONDS, flat, precision="bf16x3", for_training=False)
    big = next(i for i, m in enumerate(mols) if packing.choose_bucket(m["graph"]) == len(packing.DEFAULT_BUCKET_SIZES) - 1)
    with pytest.raises(GgnnError, match=r"graph_ids\[1\] = %d: graph of \d+ nodes does not fit nodes_per_graph = 8" % big) as ex:
        ds.prepare_batch([len(mols) - 5, big], save_for_backward=False, nodes_per_graph=8)   # a 3-node hand-made graph fits, the big one not
    assert ex.value.code == -1   # GGNN_EINVAL
    # the sparse call on a dense dataset (DeviceDataset.prepare_batch always takes the dense call for one)
    h, ids = C.c_void_p(), np.zeros(1, np.int64)
    assert ds.lib.ggnn_dataset_prepare_batch(ds._h, 0, ids.ctypes.data, 1, C.byref(h)) == -1   # GGNN_EINVAL
    assert "prepared with ggnn_dataset_prepare_batch_dense" in ds.lib.ggnn_dataset_batch_error(h).decode()
    ds.lib.ggnn_free_dataset_batch(h)
    with pytest.raises(GgnnError, match="nodes_per_graph = 0") as ex:
        ds.prepare_batch([0], save_for_backward=False)
    assert ex.value.code == -1
    with pytest.raises(GgnnError, match="created for training") as ex:
        ds.prepare_batch([0], save_for_backward=True, nodes_per_graph=29)
    assert ex.value.code == -3   # GGNN_ESTATE

    # the dense call on a sparse and on a GCN dataset
    from tests.test_device_data_cpu import GRU, T, gcn_graph_set, sparse_graph_set
    sparse = DeviceDataset.host_only(dict(GRU, hidden_size=100), T, packing.FlatSparseGraphs(sparse_graph_set(8), T), precision="bf16x3")
    gcn = DeviceDataset.host_only_gcn(64, 2, packing.FlatGCNGraphs(gcn_graph_set(4)))
    for other in (sparse, gcn):
        with pytest.raises(GgnnError, match="needs a dataset made by ggnn_dataset_create_dense") as ex:
            other.prepare_batch([0], nodes_per_graph=29)
        assert ex.value.code == -1

    # bad triples: the graph and the edge are named
    for bad, what in (([0, 5, 1], "bond type"), ([0, 0, 1], "bond type 0"), ([-1, 1, 1], "negative source"), ([0, 1, -2], "negative target")):
        broken = [dict(m) for m in mols[:4]]
        broken[2] = dict(broken[2], graph=broken[2]["graph"] + [bad])
        k = len(broken[2]["graph"]) - 1
        with pytest.raises(GgnnError, match=r"graph 2: edge %d = \(%d, %d, %d\) is out of range" % (k, bad[0], bad[1], bad[2])) as ex:
            DeviceDataset.host_only_dense(p, BONDS, flat_of(broken, True))
        assert ex.value.code == -5, what   # GGNN_ERANGE
    untied = [dict(m) for m in mols[:4]]
    untied[1] = dict(untied[1], graph=untied[1]["graph"] + [[0, BONDS + 1, 1]])   # its reverse type would be 2 * BONDS: past T
    with pytest.raises(GgnnError, match="graph 1: edge") as ex:
        DeviceDataset.host_only_dense(p, 2 * BONDS, flat_of(untied, False))
    assert ex.value.code == -5
    with pytest.raises(GgnnError, match="attention exists only in the sparse model") as ex:
        DeviceDataset.host_only_dense(dict(p, use_propagation_attention=True), BONDS, flat, precision="fp32")
    assert ex.value.code == -4   # GGNN_EUNSUPPORTED


def test_device_data_option_on_the_dense_model(tmp_path):
    """--device-data on DenseGGNNChemModel: params (what a checkpoint must match) do not change, and a CPU device is refused."""
    from gated_graph_neural_network_samples_b200 import chem_dense
    mols = synthetic.make_molecules(8, seed=1)
    args = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:6], "--valid_data": mols[6:], "--config": {"hidden_size": 16}}
    model = chem_dense.DenseGGNNChemModel
    assert model._resolve_params(dict(args, **{"--device-data": True})) == model._resolve_params(args)
    with pytest.raises(Exception, match="--device-data .* needs a CUDA device"):
        model(dict(args, **{"--device-data": True}))
