"""GPU: sparse batches built on the device from CUDA adjacency lists (``set_graph_sparse_device``, DESIGN 2.15).

The host builder is the oracle: for the same lists, the device build must leave the engine with ``prepare_graph_sparse`` (or
``prepare_graph_sparse_weighted``) + ``set_graph_prepared``'s plan text, message count and graph image, every byte included.  Covered:

1. bytes at hidden 24 / 100 / 128 / 256 / 512, fp32 / bf16x3 / bf16, save_for_backward on and off, attention on the fp32 kernels and on the
   tensor cores, CudnnCompatibleGRUCell on the tensor cores, message-weighted and not; on cfg2's molecules, the 100 000-node batch, a
   component over 128 rows, a cfg5-like single graph, the edge-case batch (empty type, isolated nodes, self-loops, duplicates), V = 0,
   T = 1, T = 32 and T = 16 with attention;
2. the forward and every gradient (d h0, the weights', d message_weights) bit-identical to the host-built batch, in deterministic mode;
3. two device builds give one image, and the NULL in-degree table equals the packer's;
4. refusals with the host builder's code and text, and GGNN_ESTATE for a forward after one;
5. one engine alternating device-built, host-prepared and dataset batches, each forward against float64;
6. guard bands around the caller's lists and in-degree table;
7. a SparseGGNNChemModel training step with CUDA adjacency feeds against the host feeds.
"""
import collections

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import workloads
from gated_graph_neural_network_samples_b200.engine import GgnnError, PropagationEngine
from oracle import ggnn_oracle as O
from tests import _util as U
from tests import test_canaries_cpu as K
from tests import test_gpu_message_weights as MWT

pytestmark = pytest.mark.gpu

def _codes():
    """The GGNN_E* values of the header (read, not assumed)."""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "ggnn_b200.h")) as f:
        return {k: int(v) for k, v in re.findall(r"(GGNN_E[A-Z]+)\s*=\s*(-?\d+)", f.read())}


CODES = _codes()


# ---------------------------------------------------------------------------------------------------------------- batches
def _indeg(adj, V, T):
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return indeg


def _random_graph(V, E, T, seed):
    rng = np.random.default_rng(seed)
    adj = [np.stack([rng.integers(0, V, E), rng.integers(0, V, E)], 1).astype(np.int32) for _ in range(T)]
    return adj, _indeg(adj, V, T)


def _workload(name):
    wl = workloads.build(name)
    adj = [np.asarray(a, np.int32).reshape(-1, 2) for a in wl["adjacency_lists"]]
    return adj, np.asarray(wl["num_incoming_edges_per_type"], np.float32)


def batch(kind, T):
    """(adjacency lists, in-degree table) of a batch kind."""
    if kind == "cfg2":
        return _workload("cfg2")
    if kind == "100k":
        return _workload("default_batch_100k_nodes")
    if kind == "cfg5":
        return _workload("cfg5_rgcn")
    if kind in ("big", "edges", "mol"):
        adj, indeg, _ = MWT.make_batch(kind, 8, T)
        return adj, indeg
    if kind == "empty":
        return [np.zeros((0, 2), np.int32) for _ in range(T)], np.zeros((0, T), np.float32)
    if kind == "rand":   # every edge type present, components of all sizes
        return _random_graph(600, 300, T, seed=T)
    raise KeyError(kind)


def _cuda_lists(adj):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a, np.int32).reshape(-1, 2)).cuda() for a in adj]


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


# ---------------------------------------------------------------------------------------------------------------- engines
Cfg = collections.namedtuple("Cfg", "D precision att att_tc cudnn T")


def cfg(D, precision, att=False, att_tc=False, cudnn=False, T=4):
    return Cfg(D, precision, att, att_tc, cudnn, T)


def params_of(c):
    return {"hidden_size": c.D, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "use_edge_bias": True,
            "use_edge_msg_avg_aggregation": True, "graph_rnn_cell": "CudnnCompatibleGRUCell" if c.cudnn else "GRU",
            "graph_rnn_activation": "tanh", "use_propagation_attention": c.att or c.att_tc}


def engine(c):
    return PropagationEngine(params_of(c), c.T, precision=c.precision, attention_tensor_cores=c.att_tc, cudnn_gru_tensor_cores=c.cudnn)


def host_build(eng, adj, indeg, weighted):
    """The host builder's plan text, message count and image for the engine's configuration and save flag."""
    g = (eng.prepare_graph_sparse_weighted if weighted else eng.prepare_graph_sparse)(adj, indeg)
    info = g.info()
    return info["plan"], info["num_messages"], g.image(), g


def device_build(eng, adj, indeg, weighted, table=True):
    V = indeg.shape[0]
    eng.set_graph_sparse_device(V, _cuda_lists(adj), _cuda(indeg) if table else None, message_weighted=weighted)
    return eng.plan, eng.num_messages(), eng.graph_image()


def assert_same_image(got, want, tag):
    assert got.nbytes == want.nbytes, (tag, got.nbytes, want.nbytes)
    if not np.array_equal(got, want):
        diff = np.nonzero(got != want)[0]
        pytest.fail("%s: %d bytes differ, first at %d (device %d, host %d)" % (tag, diff.size, diff[0], got[diff[0]], want[diff[0]]))


# ---------------------------------------------------------------------------------------------------------------- 1. bytes
BYTE_CASES = [
    ("fp32-24", cfg(24, "fp32"), "cfg2"),
    ("fp32-100", cfg(100, "fp32"), "cfg2"),
    ("fp32-100-big", cfg(100, "fp32"), "big"),
    ("fp32-256", cfg(256, "fp32"), "cfg2"),
    ("fp32-512", cfg(512, "fp32"), "cfg2"),
    ("bf16x3-24", cfg(24, "bf16x3"), "cfg2"),
    ("bf16x3-100", cfg(100, "bf16x3"), "cfg2"),
    ("bf16x3-128", cfg(128, "bf16x3"), "cfg2"),
    ("bf16x3-100-big", cfg(100, "bf16x3"), "big"),
    ("bf16x3-256", cfg(256, "bf16x3"), "cfg2"),
    ("bf16x3-512", cfg(512, "bf16x3"), "cfg2"),
    ("bf16-100", cfg(100, "bf16"), "cfg2"),
    ("bf16-256", cfg(256, "bf16"), "cfg2"),
    ("bf16x3-100-100k", cfg(100, "bf16x3"), "100k"),
    ("bf16x3-256-100k", cfg(256, "bf16x3"), "100k"),
    ("fp32-100-cfg5", cfg(100, "fp32"), "cfg5"),
    ("bf16x3-100-cfg5", cfg(100, "bf16x3"), "cfg5"),
    ("fp32-100-edges", cfg(100, "fp32"), "edges"),
    ("bf16x3-100-edges", cfg(100, "bf16x3"), "edges"),
    ("bf16x3-256-edges", cfg(256, "bf16x3"), "edges"),
    ("fp32-100-empty", cfg(100, "fp32"), "empty"),
    ("bf16x3-256-empty", cfg(256, "bf16x3"), "empty"),
    ("bf16x3-100-t1", cfg(100, "bf16x3", T=1), "mol"),
    ("fp32-64-t32", cfg(64, "fp32", T=32), "rand"),
    ("bf16x3-256-t32", cfg(256, "bf16x3", T=32), "rand"),
    ("att-fp32-100-t16", cfg(100, "fp32", att=True, T=16), "rand"),
    ("att-tc-100-t16", cfg(100, "bf16x3", att_tc=True, T=16), "rand"),
    ("att-tc-256", cfg(256, "bf16x3", att_tc=True), "cfg2"),
    ("cudnn-tc-100", cfg(100, "bf16x3", cudnn=True), "cfg2"),
    ("cudnn-tc-256-edges", cfg(256, "bf16", cudnn=True), "edges"),
]


@pytest.mark.parametrize("name,c,kind", BYTE_CASES, ids=[b[0] for b in BYTE_CASES])
@pytest.mark.parametrize("save", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_device_image_equals_host_image(name, c, kind, save, weighted):
    if weighted and (c.att or c.att_tc):
        pytest.skip("message weights are refused with attention (test_refusals)")
    adj, indeg = batch(kind, c.T)
    eng = engine(c)
    eng.set_save_for_backward(save)
    plan, M, want, _ = host_build(eng, adj, indeg, weighted)
    got_plan, got_M, got = device_build(eng, adj, indeg, weighted)
    assert got_plan == plan, (got_plan, plan)
    assert got_M == M == sum(a.shape[0] for a in adj)
    assert_same_image(got, want, "%s save=%s weighted=%s" % (name, save, weighted))


# ---------------------------------------------------------------------------------------------------------------- 2. bits through the kernels
Bits = collections.namedtuple("Bits", "name D precision weighted batch env")
BITS = [
    Bits("ffma-local", 100, "fp32", False, "mol", {}),
    Bits("ffma-local-msgw", 100, "fp32", True, "mol", {}),
    Bits("tc-local", 100, "bf16x3", False, "mol", {}),
    Bits("tc-local-msgw", 100, "bf16x3", True, "mol", {}),
    Bits("tc-global", 100, "bf16x3", True, "big", {}),
    Bits("stream-256", 256, "bf16x3", False, "mol", {}),
    Bits("stream-256-msgw", 256, "bf16x3", True, "edges", {}),
    Bits("step-260-msgw", 260, "fp32", True, "mol", {}),
]


def _run_bits(b, device, monkeypatch):
    """Forward and backward (deterministic, bf16x3 backward on the tensor-core precisions) of batch b built on the host or the device."""
    import torch
    MWT._env(monkeypatch, b.env)
    c = MWT.case(b.name, b.D, b.precision, "", batch=b.batch)
    adj, indeg, h0 = MWT.make_batch(b.batch, b.D, c.T)
    M = sum(a.shape[0] for a in adj)
    eng = MWT.engine_for(c, det=True, bwd="bf16x3" if b.precision != "fp32" else "fp32")
    dev_w = U.to_cuda_weights(MWT.layer_weights(c))
    eng.set_weights(dev_w)
    eng.set_save_for_backward(True)
    if device:
        eng.set_graph_sparse_device(indeg.shape[0], _cuda_lists(adj), _cuda(indeg), message_weighted=b.weighted)
    else:
        g = (eng.prepare_graph_sparse_weighted if b.weighted else eng.prepare_graph_sparse)(adj, indeg)
        eng.set_graph_prepared(g)
    if b.weighted:
        eng.set_message_weights(_cuda(MWT.draw_weights(M, "signed")))
    th0 = _cuda(h0)
    out = eng.forward(th0)
    g_out = np.random.default_rng(9).normal(0, 1, out.shape).astype(np.float32)
    grads = [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in dev_w]
    dh0 = torch.zeros_like(th0)
    dmw = torch.zeros(M, dtype=torch.float32, device="cuda") if b.weighted else None
    eng.backward(_cuda(g_out), grads, dh0, d_message_weights=dmw)
    eng.sync_check()
    res = {"out": out.cpu().numpy(), "dh0": dh0.cpu().numpy(), "plan": eng.plan}
    for l, lw in enumerate(grads):
        for k, t in lw.items():
            res["d%d_%s" % (l, k)] = t.cpu().numpy()
    if dmw is not None:
        res["dmw"] = dmw.cpu().numpy()
    return res


@pytest.mark.parametrize("b", BITS, ids=[b.name for b in BITS])
def test_forward_and_gradients_bit_identical_to_host_batch(b, monkeypatch):
    host = _run_bits(b, False, monkeypatch)
    dev = _run_bits(b, True, monkeypatch)
    assert dev["plan"] == host["plan"]
    assert sorted(dev) == sorted(host)
    for k in host:
        if k != "plan":
            assert np.all(np.isfinite(dev[k])), k
            np.testing.assert_array_equal(dev[k].view(np.uint32), host[k].view(np.uint32), err_msg="%s %s" % (b.name, k))


# ---------------------------------------------------------------------------------------------------------------- 3. repeatability
@pytest.mark.parametrize("c,kind", [(cfg(100, "bf16x3"), "cfg2"), (cfg(256, "bf16x3"), "100k"), (cfg(100, "fp32"), "edges")],
                         ids=["tc-cfg2", "stream-100k", "ffma-edges"])
def test_two_device_builds_and_the_null_table(c, kind):
    adj, indeg = batch(kind, c.T)   # the packer's table (and the edge-case batch's) is the per-(target, type) message count
    assert np.array_equal(indeg, _indeg(adj, indeg.shape[0], c.T))
    eng = engine(c)
    eng.set_save_for_backward(True)
    first = device_build(eng, adj, indeg, False)[2]
    second = device_build(eng, adj, indeg, False)[2]
    null = device_build(eng, adj, indeg, False, table=False)[2]
    assert_same_image(second, first, "rebuild")
    assert_same_image(null, first, "NULL table")


# ---------------------------------------------------------------------------------------------------------------- 4. refusals
def _host_error(eng, adj, indeg, weighted=False):
    with pytest.raises(GgnnError) as h:
        host_build(eng, adj, indeg, weighted)
    return h.value


def _refusal(eng, adj, indeg, weighted=False):
    with pytest.raises(GgnnError) as d:
        eng.set_graph_sparse_device(indeg.shape[0], _cuda_lists(adj), _cuda(indeg), message_weighted=weighted)
    return d.value


@pytest.mark.parametrize("bad", [-1, "V"])
def test_out_of_range_edge_named_like_the_host_builder(bad):
    import torch
    c = cfg(100, "bf16x3")
    adj, indeg = batch("cfg2", 4)
    V = indeg.shape[0]
    adj = [a.copy() for a in adj]
    i = adj[2].shape[0] // 2
    adj[2][i, 1] = -1 if bad == -1 else V
    adj[2][i + 3, 0] = V + 5   # a later bad edge of the same type is not the one named
    adj[3][0, 0] = -7          # nor one of a later type
    eng = engine(c)
    good, _ = batch("cfg2", 4)
    eng.set_graph_sparse_device(V, _cuda_lists(good), _cuda(indeg))   # a good batch, which the refused call forgets
    host = _host_error(eng, adj, indeg)
    got = _refusal(eng, adj, indeg)
    assert got.code == CODES["GGNN_ERANGE"]
    assert str(got) == str(host), (str(got), str(host))
    assert "edge %d of type 2" % i in str(got)
    with pytest.raises(GgnnError) as f:
        eng.forward(torch.zeros(V, c.D, device="cuda"))
    assert f.value.code == CODES["GGNN_ESTATE"]


def test_message_weights_with_attention_refused():
    adj, indeg = batch("cfg2", 4)
    for c in (cfg(100, "fp32", att=True), cfg(100, "bf16x3", att_tc=True)):
        eng = engine(c)
        host = _host_error(eng, adj, indeg, weighted=True)
        got = _refusal(eng, adj, indeg, weighted=True)
        assert got.code == CODES["GGNN_EUNSUPPORTED"] and str(got) == str(host)


def test_host_tensors_and_wrong_types_raise_before_the_call():
    import torch
    c = cfg(100, "bf16x3")
    adj, indeg = batch("mol", 4)
    V = indeg.shape[0]
    eng = engine(c)
    eng.set_graph_sparse_device(V, _cuda_lists(adj), _cuda(indeg))   # a good batch, which every refusal below forgets
    lists = _cuda_lists(adj)
    bad_feeds = [
        ([a.cpu() for a in lists], None),                                   # host tensors
        ([np.asarray(a) for a in adj], None),                               # NumPy arrays
        ([a.to(torch.int64) for a in lists], None),                         # wrong dtype
        ([a.reshape(-1) for a in lists], None),                             # wrong shape
        ([a.t() for a in lists], None),                                     # not contiguous (and [2, E])
        (lists[:3], None),                                                  # wrong number of lists
        (lists, _cuda(indeg).to(torch.float64)),                            # table dtype
        (lists, _cuda(indeg)[:-1]),                                         # table shape
        (lists, torch.from_numpy(indeg)),                                   # host table
    ]
    for feeds, table in bad_feeds:
        with pytest.raises(GgnnError):
            eng.set_graph_sparse_device(V, feeds, table)
    with pytest.raises(GgnnError):
        eng.set_graph_sparse_device(-1, lists, None)
    # the library's own checks: a host pointer behind the Python checks is refused with GGNN_EINVAL
    import ctypes as C
    host = [np.ascontiguousarray(a) for a in adj]
    ptrs = (C.c_void_p * 4)(*[a.ctypes.data for a in host])
    counts = (C.c_int32 * 4)(*[a.shape[0] for a in host])
    rc = eng.lib.ggnn_set_graph_sparse_device(eng._h, V, ptrs, counts, None, 0, eng._stream())
    assert rc == CODES["GGNN_EINVAL"], rc
    with pytest.raises(GgnnError) as f:
        eng.forward(torch.zeros(V, c.D, device="cuda"))
    assert f.value.code == CODES["GGNN_ESTATE"]


# ---------------------------------------------------------------------------------------------------------------- 5. lifecycle
def test_one_engine_alternates_device_host_and_dataset_batches():
    import torch
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset
    from tests.test_device_data_cpu import T, sparse_graph_set
    c = MWT.case("life", 100, "bf16x3", "", T=T)
    w = MWT.layer_weights(c)
    p = MWT.params(c)
    eng = MWT.engine_for(c)
    eng.set_weights(U.to_cuda_weights(w))
    flat = packing.FlatSparseGraphs(sparse_graph_set(), T)
    ds = DeviceDataset.for_engine(eng, flat, for_training=False)
    order = ["device", "host", "dataset", "device-msgw", "device", "dataset", "host", "device"]
    for k, kind in enumerate(order):
        adj, indeg, h0 = MWT.make_batch(["mol", "edges", "big"][k % 3], c.D, c.T, seed=k)
        mw = None
        if kind == "dataset":
            ids = np.arange(flat.num_graphs)[k::3]
            th0, _, _ = eng.set_graph_from_dataset(ds.prepare_batch(ids, save_for_backward=False))
            packed = flat.pack(ids, c.D)
            adj, indeg, h0 = packed["adjacency_lists"], packed["num_incoming_edges_per_type"], th0.cpu().numpy()
        elif kind == "host":
            eng.set_graph_prepared(eng.prepare_graph_sparse(adj, indeg))
        elif kind == "device":
            eng.set_graph_sparse_device(indeg.shape[0], _cuda_lists(adj), _cuda(indeg))
        else:
            eng.set_graph_sparse_device(indeg.shape[0], _cuda_lists(adj), None, message_weighted=True)
            with pytest.raises(GgnnError) as f:   # a message-weighted batch needs its weights first
                eng.forward(_cuda(h0))
            assert f.value.code == CODES["GGNN_ESTATE"]
            mw = MWT.draw_weights(sum(a.shape[0] for a in adj), "signed", seed=k)
            eng.set_message_weights(_cuda(mw))
        out = eng.forward(_cuda(h0)).cpu().numpy()
        eng.sync_check()
        if mw is None:
            ref = O.sparse_propagation_loops(h0, adj, indeg, w, p)
        else:
            ref = MWT.MW.propagation_torch(h0, adj, indeg, w, p, mw, dtype=torch.float64).numpy()
        err = U.max_rel_err(out, ref)
        print("\nDEVGRAPH lifecycle %-12s %.2e  %s" % (kind, err, eng.plan))
        assert np.all(np.isfinite(out)) and err < 1e-4, (k, kind, err, eng.plan)


# ---------------------------------------------------------------------------------------------------------------- 6. canaries
@pytest.mark.parametrize("c,kind", [(cfg(100, "bf16x3"), "edges"), (cfg(256, "bf16x3"), "big"), (cfg(100, "fp32"), "mol")],
                         ids=["tc-edges", "stream-big", "ffma-mol"])
def test_guard_bands_around_the_lists_and_the_table_stay_unread(c, kind):
    """Every list and the in-degree table sit between two bands of payload words (as edges: node ids far out of range; as in-degrees:
    NaN).  A read of a band would be refused or show in the image: the image is the host builder's and the bands are untouched."""
    adj, indeg = batch(kind, c.T)
    eng = engine(c)
    eng.set_save_for_backward(True)
    _, _, want, _ = host_build(eng, adj, indeg, False)
    bands, lists = [], []
    for a in adj:
        g = K.guarded(max(a.size, 1))
        ints = g.view.view(__import__("torch").int32)
        if a.size:
            ints[:a.size].copy_(_cuda_lists([a])[0].reshape(-1))
        lists.append(ints[:a.size].reshape(-1, 2))
        bands.append(g)
    gt = K.guarded(max(indeg.size, 1))
    gt.view[:indeg.size].copy_(_cuda(indeg).reshape(-1))
    bands.append(gt)
    eng.set_graph_sparse_device(indeg.shape[0], lists, gt.view[:indeg.size].reshape(indeg.shape))
    assert_same_image(eng.graph_image(), want, "guarded")
    assert all(g.bands_intact() for g in bands)


# ---------------------------------------------------------------------------------------------------------------- 7. the plug-in
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_plugin_training_step_with_cuda_adjacency_feeds(tmp_path, precision):
    """One SparseGGNNChemModel step in deterministic mode: CUDA adjacency lists give the host feed's loss and gradients, bit for bit."""
    import torch
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    mols = synthetic.make_molecules(64, seed=5, num_bond_types=4)
    m = SparseGGNNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:48], "--valid_data": mols[48:],
                             "--config": dict(hidden_size=32, layer_timesteps=[2, 1], residual_connections={"1": [0]}, use_edge_bias=True,
                                              batch_size=400, random_seed=3)})
    m.make_train_step()
    feed = dict(next(iter(m.make_minibatch_iterator(m.train_data, True))))
    feed.pop("_prepared_graph", None)
    for k in ("graph_state_keep_prob", "edge_weight_dropout_keep_prob", "out_layer_dropout_keep_prob"):
        feed[m.placeholders.get(k, k)] = 1.0
    variables = [v for _, v in m.graph_model_variables()]
    keys = m.placeholders["adjacency_lists"]
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)   # the engine's fixed-order sums; torch's own ops only warn
    try:
        results = []
        for device in (False, True):
            f = dict(feed)
            if device:
                f.update({k: torch.from_numpy(np.asarray(f[k], np.int32).reshape(-1, 2)).cuda() for k in keys})
            loss = m.forward_batch(f)[0]
            grads = torch.autograd.grad(loss, variables)
            results.append((float(loss), [g.cpu().numpy() for g in grads], m.engine.plan))
    finally:
        torch.use_deterministic_algorithms(was)
    (lh, gh, ph), (ld, gd, pd) = results
    assert pd == ph and ld == lh, (ld, lh)
    for a, b in zip(gd, gh):
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))
