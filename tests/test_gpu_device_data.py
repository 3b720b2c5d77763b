"""GPU: batches assembled on the device from a ``DeviceDataset`` are the batches the packers feed.

For GGNN (LOCAL, GLOBAL, streaming, attention) and GCN engines, with and without save_for_backward, and for a batch taken after a larger one
(so that every buffer is reused): the device-built graph image is byte-identical to ``PreparedGraph.image`` of the same batch built from its
wire format; h0, targets, mask and the readout map equal the packer's; the forward and d h0 are bit-identical to the feed-dict path."""
import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing
from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GCNEngine, GgnnError, PreparedGraph, PropagationEngine, weight_shapes
from tests.test_device_data_cpu import GRU, T, batch_ids, gcn_graph_set, sparse_graph_set

pytestmark = pytest.mark.gpu


def _weights(params, L, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    out = []
    for l in range(L):
        out.append({k: (torch.rand(s, generator=g) * 0.2 - 0.1).cuda().contiguous() for k, s in weight_shapes(params, T, l).items()})
    return out


def _readout(eng, h, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    D = eng.D
    ws = [(torch.rand(n, generator=g) - 0.5).cuda() for n in (2 * D, 1, D, 1)]
    return eng.readout_forward(h, h, *ws)


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _batches(N):
    """A large batch first (buffers grow), then the seeded batches, smaller ones after larger."""
    return [np.arange(N)[::-1].copy()] + batch_ids(N, seed=7)


def _check_batch(eng, b, packed, ref_graph, save, seed):
    import torch
    h0, tv, tm = eng.set_graph_from_dataset(b)
    got, want = eng.graph_image(), ref_graph.image()
    assert got.shape == want.shape
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:32]
    if b.G == 0:
        return
    np.testing.assert_array_equal(h0.cpu().numpy(), packed["initial_node_representation"])
    np.testing.assert_array_equal(tv.cpu().numpy(), packed["target_values"])
    np.testing.assert_array_equal(tm.cpu().numpy(), packed["target_mask"])
    out_ds = eng.forward(h0)
    ro_ds = _readout(eng, out_ds, seed)
    d_ds = None
    if save:
        d_ds = torch.zeros_like(h0)
        for g in eng._grads:
            for v in g.values():
                v.zero_()
        eng.backward(torch.ones_like(out_ds), eng._grads, d_ds)
        g_ds = [{k: v.clone() for k, v in g.items()} for g in eng._grads]
    # the same batch through the feed-dict path
    eng.set_graph_prepared(ref_graph)
    eng.readout_set_graphs(b.G, packed["graph_nodes_list"])
    h0_ref = torch.from_numpy(packed["initial_node_representation"]).cuda()
    out_ref = eng.forward(h0_ref)
    assert torch.equal(out_ds, out_ref)
    assert torch.equal(ro_ds, _readout(eng, out_ref, seed))
    if save:   # deterministic mode: d h0 and every weight gradient bit for bit
        d_ref = torch.zeros_like(h0_ref)
        for g in eng._grads:
            for v in g.values():
                v.zero_()
        eng.backward(torch.ones_like(out_ref), eng._grads, d_ref)
        assert torch.equal(d_ds, d_ref)
        for l, (a, b) in enumerate(zip(g_ds, eng._grads)):
            for k in a:
                assert torch.equal(a[k], b[k]), (l, k)


SPARSE = [  # hidden, precision, attention
    (100, "bf16x3", False), (256, "bf16x3", False), (100, "fp32", False), (64, "fp32", True)]


@pytest.mark.parametrize("hidden,precision,att", SPARSE)
@pytest.mark.parametrize("save", [False, True])
def test_sparse_dataset_batches_match_the_feed_dict_path(hidden, precision, att, save):
    import torch
    flat = packing.FlatSparseGraphs(sparse_graph_set(), T)
    params = dict(GRU, hidden_size=hidden, use_propagation_attention=att)
    eng = PropagationEngine(params, T, precision=precision)
    w = _weights(params, 2, hidden)
    eng.set_weights(w)
    eng.set_save_for_backward(save)
    eng.set_deterministic(True)
    eng._grads = [{k: torch.zeros_like(v) for k, v in l.items()} for l in w]
    ds = DeviceDataset.for_engine(eng, flat, for_training=save)
    for i, ids in enumerate(_batches(flat.num_graphs)):
        b = ds.prepare_batch(ids, save_for_backward=save)
        packed = flat.pack(ids, hidden) if len(ids) else None
        # the reference is built in plain host memory: a fresh one is zero in the alignment gaps, as the device image is
        adj, indeg = ((packed["adjacency_lists"], packed["num_incoming_edges_per_type"]) if packed is not None
                      else ([np.zeros((0, 2), np.int32)] * T, np.zeros((0, T), np.float32)))
        ref = PreparedGraph.host_only(params, T, adj, indeg, precision=precision, num_sms=_sms(), save_for_backward=save)
        _check_batch(eng, b, packed, ref, save, i)
    eng.sync_check()


@pytest.mark.parametrize("hidden,precision", [(100, "bf16x3"), (64, "fp32")])
@pytest.mark.parametrize("save", [False, True])
def test_gcn_dataset_batches_match_the_feed_dict_path(hidden, precision, save):
    import torch
    flat = packing.FlatGCNGraphs(gcn_graph_set())
    eng = GCNEngine(hidden, 3, use_bias=True, precision=precision)
    g = torch.Generator().manual_seed(hidden)
    ks = [(torch.rand(hidden, hidden, generator=g) * 0.2 - 0.1).cuda() for _ in range(3)]
    bs = [(torch.rand(hidden, generator=g) * 0.2 - 0.1).cuda() for _ in range(3)]
    eng.set_weights(ks, bs)
    eng.set_save_for_backward(save)
    eng.set_deterministic(True)
    eng._grads = [{"kernel": torch.zeros_like(k), "bias": torch.zeros_like(b)} for k, b in zip(ks, bs)]
    ds = DeviceDataset.for_engine(eng, flat, for_training=save)
    for i, ids in enumerate(_batches(flat.num_graphs)):
        b = ds.prepare_batch(ids, save_for_backward=save)
        packed = flat.pack(ids, hidden) if len(ids) else None
        V, lst, w = ((packed["initial_node_representation"].shape[0], packed["adjacency_list"], packed["adjacency_weights"]) if packed is not None
                     else (0, np.zeros((0, 2), np.int64), np.zeros(0)))
        ref = PreparedGraph.host_only_gcn(hidden, 3, V, lst, w, use_bias=True, precision=precision, num_sms=_sms(), save_for_backward=save)
        _check_batch(eng, b, packed, ref, save, i)
    eng.sync_check()


def test_lifetime_and_refusals():
    import torch
    flat = packing.FlatSparseGraphs(sparse_graph_set(20), T)
    params = dict(GRU, hidden_size=100)
    eng = PropagationEngine(params, T, precision="bf16x3")
    w = _weights(params, 2, 1)
    eng.set_weights(w)
    eng.set_save_for_backward(True)
    grads = [{k: torch.zeros_like(v) for k, v in l.items()} for l in w]
    ds = DeviceDataset.for_engine(eng, flat)
    # dataset batch -> feed-dict batch -> dataset batch on one engine: each forward is the one of its batch
    ids = np.array([4, 2, 9])
    packed = flat.pack(ids, 100)
    h0, _, _ = eng.set_graph_from_dataset(ds.prepare_batch(ids))
    out1 = eng.forward(h0).clone()
    eng.set_graph_sparse(packed["adjacency_lists"], packed["num_incoming_edges_per_type"])
    assert torch.equal(eng.forward(torch.from_numpy(packed["initial_node_representation"]).cuda()), out1)
    h0, _, _ = eng.set_graph_from_dataset(ds.prepare_batch(ids))
    assert torch.equal(eng.forward(h0), out1)
    # a new batch forgets the last forward: layer_state, backward and the readout map of the previous one are refused
    eng.set_graph_from_dataset(ds.prepare_batch([1]))
    with pytest.raises(GgnnError):
        eng.layer_state(1)
    with pytest.raises(GgnnError):
        eng.backward(torch.ones_like(out1), grads, None)
    # a dataset made for one engine shape is refused by another
    other = PropagationEngine(dict(params, hidden_size=64), T, precision="bf16x3")
    with pytest.raises(GgnnError, match="different engine configuration") as ex:
        other.set_graph_from_dataset(ds.prepare_batch([0]))
    assert ex.value.code == -1   # GGNN_EINVAL
    gcn = GCNEngine(100, 2, precision="bf16x3")
    with pytest.raises(GgnnError, match="GGNN engine") as ex:
        gcn.set_graph_from_dataset(ds.prepare_batch([0]))
    assert ex.value.code == -3   # GGNN_ESTATE
    eng.sync_check()
