"""GPU: the readout map built from CUDA arrays (``readout_set_graphs`` with CUDA tensors, ``ggnn_readout_set_graphs_device``, DESIGN 2.17).

The host builder is the oracle: for the same list or mask, the device build must leave the engine with the host map, section by section.
Covered:

1. sections through ``ggnn_readout_map``: the packer's grouped lists of cfg2 and of the 100 000-node batch, shuffled lists (the stable
   by-graph permutation), leading / interior / trailing empty graphs, G = 1, V = 0, G = 0 with V = 0, and dense maps with a mask
   (b = 0 included) and without one;
2. ``readout_forward``, ``readout_backward`` and ``readout_predict`` over the two maps: the same bits in deterministic mode; in atomic mode
   the same bits on grouped lists (weight gradients, summed with atomics in that mode, at fp32 tolerance) and fp32 tolerance on shuffled
   ones;
3. refusals with the host builder's code and text, and no map left behind by a refused call;
4. one engine alternating graph uploads, host maps, device maps and dataset batches, each equal to a fresh engine's;
5. guard bands around the caller's list and mask;
6. one training step of each plug-in with every array of the feed a CUDA tensor, against the host feed, bit for bit.
"""
import functools

import numpy as np
import pytest

from tests import test_canaries_cpu as K

pytestmark = pytest.mark.gpu

D = 32


def _codes():
    """The GGNN_E* values of the header (read, not assumed)."""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "ggnn_b200.h")) as f:
        return {k: int(v) for k, v in re.findall(r"(GGNN_E[A-Z]+)\s*=\s*(-?\d+)", f.read())}


CODES = _codes()


def _engine(det=True):
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine({"hidden_size": D, "layer_timesteps": [1], "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}, 4)
    eng.set_deterministic(det)
    return eng


def _cuda(a, dtype=np.float32):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------- cases
@functools.lru_cache(maxsize=None)
def _workload_list(name):
    from gated_graph_neural_network_samples_b200 import workloads
    w = workloads.build(name)
    return int(w["num_graphs"]), np.asarray(w["graph_nodes_list"], np.int32)


def sparse_case(kind):
    """(G, graph_nodes_list int32 [V])."""
    rng = np.random.default_rng(7)
    if kind == "cfg2":
        return _workload_list("cfg2")
    if kind == "100k":
        return _workload_list("default_batch_100k_nodes")
    if kind == "shuffled":
        G, gnl = _workload_list("cfg2")
        return G, rng.permutation(gnl).astype(np.int32)
    if kind == "shuffled-100k":
        G, gnl = _workload_list("default_batch_100k_nodes")
        return G, rng.permutation(gnl).astype(np.int32)
    if kind == "one-descent":      # grouped but for one node at the end
        G, gnl = _workload_list("cfg2")
        gnl = gnl.copy()
        gnl[-1] = 0
        return G, gnl
    sizes = np.array([0, 0, 3, 0, 5, 1, 0, 0, 2, 0, 0])   # leading, interior and trailing empty graphs
    if kind == "empty-graphs":
        return len(sizes), np.repeat(np.arange(len(sizes), dtype=np.int32), sizes)
    if kind == "empty-graphs-shuffled":
        return len(sizes), rng.permutation(np.repeat(np.arange(len(sizes), dtype=np.int32), sizes)).astype(np.int32)
    if kind == "G1":
        return 1, np.zeros(9, np.int32)
    if kind == "V0":
        return 4, np.zeros(0, np.int32)
    if kind == "G0V0":
        return 0, np.zeros(0, np.int32)
    raise KeyError(kind)


SPARSE = ["cfg2", "100k", "shuffled", "shuffled-100k", "one-descent", "empty-graphs", "empty-graphs-shuffled", "G1", "V0", "G0V0"]
GROUPED = {"cfg2", "100k", "empty-graphs", "G1", "V0", "G0V0"}


def dense_case(kind):
    """(b, v, node_mask float32 [b, v])."""
    rng = np.random.default_rng(9)
    b, v = {"b9v16": (9, 16), "cfg-bucket": (256, 29), "b1v1": (1, 1), "b0": (0, 5)}[kind]
    return b, v, (rng.random((b, v)) < 0.7).astype(np.float32)


DENSE = ["b9v16", "cfg-bucket", "b1v1", "b0"]


def assert_same_map(got, want, tag):
    np.testing.assert_array_equal(got["graph_of"], want["graph_of"], err_msg=tag + " graph_of")
    np.testing.assert_array_equal(got["start"], want["start"], err_msg=tag + " start")
    assert got["grouped"] == want["grouped"], tag
    if want["perm"] is None:
        assert got["perm"] is None, tag
    else:
        np.testing.assert_array_equal(got["perm"], want["perm"], err_msg=tag + " perm")
    if want["node_mask"] is None:
        assert got["node_mask"] is None, tag
    else:
        np.testing.assert_array_equal(_bits(got["node_mask"]), _bits(want["node_mask"]), err_msg=tag + " mask")


# ---------------------------------------------------------------------------------------------------------------- 1. sections
@pytest.mark.parametrize("kind", SPARSE)
def test_sparse_map_sections_equal_the_host_builder(kind):
    G, gnl = sparse_case(kind)
    eng = _engine()
    eng.readout_set_graphs(G, graph_nodes_list=gnl)
    want = eng.readout_map()
    assert want["grouped"] == (kind in GROUPED), kind
    eng.readout_set_graphs(G, graph_nodes_list=_cuda(gnl, np.int32))
    got = eng.readout_map()
    assert_same_map(got, want, kind)
    assert got["start"][-1] == gnl.shape[0]
    eng.readout_set_graphs(G, graph_nodes_list=_cuda(gnl, np.int32))   # a second build on the same engine
    assert_same_map(eng.readout_map(), want, kind + " rebuild")
    # with a mask next to the list (the host call takes one too)
    mask = np.random.default_rng(1).random(gnl.shape[0]).astype(np.float32)
    eng.readout_set_graphs(G, graph_nodes_list=gnl, node_mask=mask)
    want = eng.readout_map()
    eng.readout_set_graphs(G, graph_nodes_list=_cuda(gnl, np.int32), node_mask=_cuda(mask))
    assert_same_map(eng.readout_map(), want, kind + " masked")


@pytest.mark.parametrize("kind", DENSE)
def test_dense_map_sections_equal_the_host_builder(kind):
    b, v, mask = dense_case(kind)
    eng = _engine()
    eng.readout_set_graphs(b, nodes_per_graph=v, node_mask=mask)
    want = eng.readout_map()
    eng.readout_set_graphs(b, nodes_per_graph=v, node_mask=_cuda(mask))
    got = eng.readout_map()
    assert_same_map(got, want, kind)
    assert got["grouped"] and got["node_mask"] is not None
    # no mask: only through the C entry (Python routes on a CUDA argument)
    lib, h, st = eng.lib, eng._h, eng._stream()
    assert lib.ggnn_readout_set_graphs(h, b * v, None, b, v, None, st) == 0
    want = eng.readout_map()
    assert lib.ggnn_readout_set_graphs_device(h, b * v, None, b, v, None, st) == 0
    got = eng.readout_map()
    assert_same_map(got, want, kind + " no mask")
    assert got["node_mask"] is None


# ---------------------------------------------------------------------------------------------------------------- 2. readout bits
def _readout_all(eng, V, G, seed=3):
    """forward, backward (d_h and the four weight gradients) and a two-task predict over the current map."""
    import torch
    rng = np.random.default_rng(seed)
    h_last, h0 = _cuda(rng.normal(0, 0.5, (V, D))), _cuda(rng.normal(0, 0.5, (V, D)))
    tasks = [tuple(_cuda(rng.normal(0, 0.3, n)) for n in (2 * D, 1, D, 1)) for _ in range(2)]
    d_out = _cuda(rng.normal(size=G))
    if G == 0:
        return []
    out = eng.readout_forward(h_last, h0, *tasks[0])
    grads = eng.readout_backward(h_last, h0, *tasks[0], d_out)
    pred = eng.readout_predict(h_last, h0, tasks)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in (out, *grads, pred)]


NAMES = ["forward", "d h_last", "d w_gate", "d b_gate", "d w_trans", "d b_trans", "predict"]


@pytest.mark.parametrize("det", [True, False], ids=["deterministic", "atomic"])
@pytest.mark.parametrize("kind", SPARSE + ["dense-" + k for k in DENSE])
def test_readout_over_the_device_map_gives_the_host_maps_bits(kind, det):
    eng = _engine(det)
    if kind.startswith("dense-"):
        b, v, mask = dense_case(kind[len("dense-"):])
        V, G, grouped = b * v, b, True
        host = dict(nodes_per_graph=v, node_mask=mask)
        dev = dict(nodes_per_graph=v, node_mask=_cuda(mask))
    else:
        G, gnl = sparse_case(kind)
        V, grouped = gnl.shape[0], kind in GROUPED
        host, dev = dict(graph_nodes_list=gnl), dict(graph_nodes_list=_cuda(gnl, np.int32))
    eng.readout_set_graphs(G, **host)
    want = _readout_all(eng, V, G)
    eng.readout_set_graphs(G, **dev)
    got = _readout_all(eng, V, G)
    for name, a, b in zip(NAMES, got, want):
        tag = "%s %s %s" % (kind, "det" if det else "atomic", name)
        exact = det or (grouped and name in ("forward", "predict", "d h_last"))
        if exact:
            np.testing.assert_array_equal(_bits(a), _bits(b), err_msg=tag)
        else:   # the atomic kernels of both maps: fp32 sums in another order
            err = float(np.max(np.abs(a - b))) / max(float(np.max(np.abs(b))), 1e-12)
            assert err < 1e-5, (tag, err)


# ---------------------------------------------------------------------------------------------------------------- 3. refusals
def _assert_no_map(eng):
    """Every readout call refuses with GGNN_ESTATE (the library's first check, ahead of its arguments')."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    z = torch.zeros(4 * D, device="cuda")
    p, st = z.data_ptr(), eng._stream()
    assert eng.lib.ggnn_readout_forward(eng._h, *([p] * 7), st) == CODES["GGNN_ESTATE"]
    assert eng.lib.ggnn_readout_backward(eng._h, *([p] * 12), st) == CODES["GGNN_ESTATE"]
    tasks = eng._readout_tasks([(z[:2 * D], z[:1], z[:D], z[:1])])
    assert eng.lib.ggnn_readout_predict(eng._h, p, p, 1, tasks, None, 1, p, st) == CODES["GGNN_ESTATE"]
    with pytest.raises(GgnnError) as f:
        eng.readout_map()
    assert f.value.code == CODES["GGNN_ESTATE"]


BAD = {
    "negative": [(1234, -1)],
    "equal-G": [(777, "G")],
    # the lowest index, not the first thread that saw one: a grid-stride thread with a low id reaches entries far down the list on its
    # later iterations, after higher ids have seen earlier ones
    "several": [(90000, -7), (20000, "G"), (60000, 2 ** 31 - 1), ("last", -1), (20001, -2)],
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_lowest_bad_entry_named_like_the_host_builder(case):
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    G, gnl = sparse_case("100k")
    bad = gnl.copy()
    first = None
    for k, val in BAD[case]:
        k = bad.shape[0] - 1 if k == "last" else k
        bad[k] = G if val == "G" else val
        first = k if first is None else min(first, k)
    eng = _engine()
    with pytest.raises(GgnnError) as h:
        eng.readout_set_graphs(G, graph_nodes_list=bad)
    eng.readout_set_graphs(G, graph_nodes_list=_cuda(gnl, np.int32))   # a good map, which the refused call drops
    with pytest.raises(GgnnError) as d:
        eng.readout_set_graphs(G, graph_nodes_list=_cuda(bad, np.int32))
    assert d.value.code == h.value.code == CODES["GGNN_ERANGE"]
    assert str(d.value) == str(h.value), (str(d.value), str(h.value))
    assert "graph_nodes_list[%d] = %d is out of range for %d graphs" % (first, bad[first], G) in str(d.value)
    _assert_no_map(eng)


def test_library_refusals():
    G, gnl = sparse_case("cfg2")
    V = gnl.shape[0]
    eng = _engine()
    lib, h, st = eng.lib, eng._h, eng._stream()
    dl, mask = _cuda(gnl, np.int32), _cuda(np.ones(V, np.float32))
    host_list, host_mask = np.ascontiguousarray(gnl), np.ones(V, np.float32)
    calls = [
        (V, host_list.ctypes.data, G, 0, None),               # a host list
        (V, dl.data_ptr(), G, 0, host_mask.ctypes.data),      # a host mask
        (G * 4, None, G, 4, host_mask.ctypes.data),           # a host mask of a dense map
        (-1, dl.data_ptr(), G, 0, None),                      # negative sizes
        (V, dl.data_ptr(), -1, 0, None),
        (V, None, G, 3, mask.data_ptr()),                     # nodes_per_graph * G != V without a list
        (V, None, G, 0, mask.data_ptr()),
    ]
    for args in calls:
        assert lib.ggnn_readout_set_graphs(h, V, host_list.ctypes.data, G, 0, None, st) == 0   # a map to drop
        assert lib.ggnn_readout_set_graphs_device(h, *args, st) == CODES["GGNN_EINVAL"], args
        _assert_no_map(eng)
    assert lib.ggnn_readout_set_graphs_device(None, V, dl.data_ptr(), G, 0, None, st) == CODES["GGNN_EINVAL"]


# ---------------------------------------------------------------------------------------------------------------- 4. lifecycle
def test_one_engine_alternates_uploads_host_maps_device_maps_and_dataset_batches():
    import torch
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset
    from tests import _util as U
    from tests.test_device_data_cpu import sparse_graph_set
    flat = packing.FlatSparseGraphs(sparse_graph_set(), 4)
    _, mb = U.molecule_batch(30, D, seed=4)
    Gs, gs = sparse_case("shuffled")
    Gg, gg = sparse_case("cfg2")
    b, v, mask = dense_case("b9v16")
    ids = np.arange(flat.num_graphs)

    def upload(eng):   # a graph upload drops the map: the readout refuses until a new one is set
        eng.set_graph_sparse(mb["adjacency_lists"], mb["num_incoming_edges_per_type"])
        _assert_no_map(eng)
        eng.readout_set_graphs(30, graph_nodes_list=_cuda(mb["graph_nodes_list"], np.int32))
        return mb["graph_nodes_list"].shape[0], 30

    def host(G, gnl=None, npg=0, m=None):
        def step(eng):
            eng.readout_set_graphs(G, graph_nodes_list=gnl, nodes_per_graph=npg, node_mask=m)
            return (gnl.shape[0] if gnl is not None else G * npg), G
        return step

    def device(G, gnl=None, npg=0, m=None):
        def step(eng):
            eng.readout_set_graphs(G, graph_nodes_list=None if gnl is None else _cuda(gnl, np.int32), nodes_per_graph=npg,
                                   node_mask=None if m is None else _cuda(m))
            return (gnl.shape[0] if gnl is not None else G * npg), G
        return step

    def dataset(sel):
        def step(eng):
            if not hasattr(eng, "test_dataset"):
                eng.test_dataset = DeviceDataset.for_engine(eng, flat, for_training=False)
            bt = eng.test_dataset.prepare_batch(sel, save_for_backward=False)
            eng.set_graph_from_dataset(bt)
            eng.test_batch = bt
            return bt.V, bt.G
        return step

    steps = [device(Gg, gg), upload, host(Gs, gs), device(Gs, gs), dataset(ids[::3]), device(b, npg=v, m=mask), host(Gg, gg),
             dataset(ids[1::2]), device(Gs, gs), upload, device(Gg, gg), host(b, npg=v, m=mask), device(Gs, gs)]
    shared = _engine()
    for k, step in enumerate(steps):
        outs, maps = [], []
        for eng in (shared, _engine()):
            V, G = step(eng)
            maps.append(eng.readout_map())
            outs.append(_readout_all(eng, V, G, seed=k))
        assert_same_map(maps[0], maps[1], "step %d" % k)
        for name, a, c in zip(NAMES, *outs):
            np.testing.assert_array_equal(_bits(a), _bits(c), err_msg="step %d %s" % (k, name))
        torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------- 5. canaries
@pytest.mark.parametrize("kind", ["cfg2", "shuffled", "empty-graphs-shuffled"])
def test_guard_bands_around_the_list_and_the_mask_stay_unread(kind):
    """The list and the mask sit between two bands of payload words: as graph ids far out of range (a read of one would be refused), as
    NaN mask entries (a read of one would show in the map).  The build succeeds, the map is the host builder's and the bands are
    untouched."""
    import torch
    G, gnl = sparse_case(kind)
    V = gnl.shape[0]
    mask = np.random.default_rng(2).random(V).astype(np.float32)
    eng = _engine()
    eng.readout_set_graphs(G, graph_nodes_list=gnl, node_mask=mask)
    want = eng.readout_map()
    gl, gm = K.guarded(V), K.guarded(V)
    ints = gl.view.view(torch.int32)
    ints.copy_(_cuda(gnl, np.int32))
    gm.view.copy_(_cuda(mask))
    eng.readout_set_graphs(G, graph_nodes_list=ints, node_mask=gm.view)
    assert_same_map(eng.readout_map(), want, "guarded " + kind)
    assert gl.bands_intact() and gm.bands_intact()


def test_guard_bands_around_a_dense_mask_stay_unread():
    b, v, mask = dense_case("cfg-bucket")
    eng = _engine()
    eng.readout_set_graphs(b, nodes_per_graph=v, node_mask=mask)
    want = eng.readout_map()
    gm = K.guarded(b * v)
    gm.view.copy_(_cuda(mask).reshape(-1))
    eng.readout_set_graphs(b, nodes_per_graph=v, node_mask=gm.view.view(b, v))
    assert_same_map(eng.readout_map(), want, "guarded dense")
    assert gm.bands_intact()


# ---------------------------------------------------------------------------------------------------------------- 6. the plug-ins
def _deterministic_step(m, feeds, variables):
    """One forward_batch + gradient per feed, in deterministic mode: [(loss, grads, plan)]."""
    import torch
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)   # the engine's fixed-order sums; torch's own ops only warn
    try:
        results = []
        for f in feeds:
            loss = m.forward_batch(dict(f))[0]
            grads = torch.autograd.grad(loss, variables)
            results.append((float(loss.detach()), [g.cpu().numpy() for g in grads], m.engine.plan))
        return results
    finally:
        torch.use_deterministic_algorithms(was)


def _assert_same_steps(results):
    (lh, gh, ph), (ld, gd, pd) = results
    assert ld == lh, (ld, lh)
    assert pd.replace(" [message-weighted]", "") == ph.replace(" [message-weighted]", ""), (pd, ph)
    assert len(gd) == len(gh)
    for a, b in zip(gd, gh):
        np.testing.assert_array_equal(_bits(a), _bits(b))


def _first_feed(m):
    feed = dict(next(iter(m.make_minibatch_iterator(m.train_data, True))))
    feed.pop("_prepared_graph", None)
    for k in ("graph_state_keep_prob", "edge_weight_dropout_keep_prob", "out_layer_dropout_keep_prob"):
        if k in m.placeholders:
            feed[m.placeholders[k]] = 1.0
    return feed


def _variables(m):
    return [v for _, v in m.trainable_variables()]


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
def test_sparse_ggnn_plugin_step_with_an_all_cuda_feed(tmp_path, bwd):
    """Every array of the feed a CUDA tensor -- adjacency lists, in-degree table, graph_nodes_list, h0, targets: the host feed's loss and
    every gradient, readout weights included, bit for bit."""
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    mols = synthetic.make_molecules(64, seed=5, num_bond_types=4)
    m = SparseGGNNChemModel({"--log_dir": str(tmp_path), "--precision": "bf16x3", "--backward-precision": bwd, "--train_data": mols[:48],
                             "--valid_data": mols[48:], "--config": dict(hidden_size=32, layer_timesteps=[2, 1], use_edge_bias=True,
                                                                         batch_size=400, random_seed=3)})
    m.make_train_step()
    feed = _first_feed(m)
    cuda = dict(feed)
    for k in m.placeholders["adjacency_lists"]:
        cuda[k] = _cuda(np.asarray(feed[k]).reshape(-1, 2), np.int32)
    cuda["graph_nodes_list"] = _cuda(feed["graph_nodes_list"], np.int32)
    for k in ("num_incoming_edges_per_type", "initial_node_representation", "target_values", "target_mask"):
        cuda[k] = _cuda(feed[k])
    _assert_same_steps(_deterministic_step(m, [feed, cuda], _variables(m)))


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
def test_sparse_gcn_plugin_step_with_an_all_cuda_feed(tmp_path, bwd):
    """adjacency_list, adjacency_weights, graph_nodes_list, h0 and targets as CUDA tensors: the host feed's loss and gradients, bit for
    bit."""
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    mols = synthetic.make_molecules(64, seed=5)
    m = SparseGCNChemModel({"--log_dir": str(tmp_path), "--precision": "bf16x3", "--backward-precision": bwd, "--train_data": mols[:48],
                            "--valid_data": mols[48:], "--config": dict(hidden_size=32, num_timesteps=3, gcn_use_bias=True, batch_size=400,
                                                                        random_seed=3)})
    m.make_train_step()
    feed = _first_feed(m)
    cuda = dict(feed)
    cuda["adjacency_list"] = _cuda(feed["adjacency_list"], np.int64)
    cuda["graph_nodes_list"] = _cuda(feed["graph_nodes_list"], np.int32)
    for k in ("adjacency_weights", "initial_node_representation", "target_values", "target_mask"):
        cuda[k] = _cuda(feed[k])
    _assert_same_steps(_deterministic_step(m, [feed, cuda], _variables(m)))


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
def test_dense_ggnn_plugin_step_with_an_all_cuda_feed(tmp_path, bwd):
    """A torch adjacency_matrix with node_mask, h0 and targets as CUDA tensors against the same adjacency with those as host arrays (a
    NumPy matrix runs another propagation plan, so the matrix is a CUDA tensor in both): the same loss and gradients, bit for bit."""
    import torch
    from gated_graph_neural_network_samples_b200 import chem_dense, synthetic
    torch.manual_seed(0)
    np.random.seed(0)
    mols = synthetic.make_molecules(64, seed=6)   # 48 training molecules fill a batch of 8 in three buckets
    m = chem_dense.DenseGGNNChemModel({"--log_dir": str(tmp_path), "--precision": "bf16x3", "--backward-precision": bwd,
                                       "--train_data": mols[:48], "--valid_data": mols[48:],
                                       "--config": {"hidden_size": 32, "batch_size": 8, "num_timesteps": 2, "random_seed": 0}})
    m.make_train_step()
    feed = _first_feed(m)
    feed["adjacency_matrix"] = _cuda(feed["adjacency_matrix"])
    cuda = dict(feed)
    for k in ("node_mask", "initial_node_representation", "target_values", "target_mask"):
        cuda[k] = _cuda(feed[k])
    _assert_same_steps(_deterministic_step(m, [feed, cuda], _variables(m)))
