"""GPU: dense batches assembled on the device from a dense ``DeviceDataset`` are the batches ``pack_dense_batch`` feeds.

For the tile-local bf16x3 kernel (hidden 100), the streaming kernels (hidden 256) and the fp32 kernel, tied and untied, with and without
save_for_backward, over one engine's sequence of batches (every bucket-29 graph at once, a small bucket, the empty batch, a large batch,
then smaller ones, the hand-made graphs, and small graphs in 30 rows each, so that streaming tiles start inside padding rows): the device-built graph image is byte-identical to ``PreparedGraph.image`` of the matrix's
batch; h0, targets, target mask and node mask equal the packer's; the forward, the fused masked readout, d h0 and every weight gradient
(deterministic mode) are bit-identical to the host-packed path."""
import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing
from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GgnnError, PreparedGraph, PropagationEngine, weight_shapes
from tests.test_dense_device_data_cpu import edge_types, flat_of, hand_made_graphs, molecules, packed, params

pytestmark = pytest.mark.gpu


def _weights(p, T, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    return [{k: (torch.rand(s, generator=g) * 0.2 - 0.1).cuda().contiguous() for k, s in weight_shapes(p, T, 0).items()}]


def _readout(eng, h, h0, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    D = eng.D
    ws = [(torch.rand(n, generator=g) - 0.5).cuda() for n in (2 * D, 1, D, 1)]
    return eng.readout_forward(h, h0, *ws)


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sequence(mols):
    """Bucket 29 at once, a small bucket, the empty batch, a large batch, smaller ones after it, the hand-made graphs (one with V_g == v)."""
    synth = len(mols) - len(hand_made_graphs())
    buckets = np.array([packing.choose_bucket(m["graph"]) for m in mols[:synth]])
    rng = np.random.default_rng(5)
    pick = lambda bk, n: rng.choice(np.flatnonzero(buckets == bk), size=n)
    sizes = packing.DEFAULT_BUCKET_SIZES
    hm = np.arange(synth, len(mols))
    return [(np.flatnonzero(buckets == len(sizes) - 1), 29), (pick(1, 7), int(sizes[1])), (np.zeros(0, np.int64), 8),
            (pick(8, 256), int(sizes[8])), (pick(8, 64), int(sizes[8])), (pick(3, 1), int(sizes[3])), (hm, 6), (hm[2:3], 6),
            (pick(0, 12), 30)]   # graphs of <= 4 nodes in 30 rows each: the streaming plan's 128-row tiles start inside padding


def _check(eng, b, pk, ref, save, seed):
    import torch
    h0, tv, tm, mask = eng.set_graph_from_dataset(b)
    got, want = eng.graph_image(), ref.image()
    assert got.shape == want.shape
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:32]
    if b.G == 0:
        return
    D = eng.D
    np.testing.assert_array_equal(h0.cpu().numpy(), pk["initial_node_representation"].reshape(-1, D))
    np.testing.assert_array_equal(tv.cpu().numpy(), pk["target_values"])
    np.testing.assert_array_equal(tm.cpu().numpy(), pk["target_mask"])
    np.testing.assert_array_equal(mask.cpu().numpy(), pk["node_mask"])
    out_ds = eng.forward(h0)
    ro_ds = _readout(eng, out_ds, h0, seed)
    if save:
        d_ds = torch.zeros_like(h0)
        for g in eng._grads:
            for v in g.values():
                v.zero_()
        eng.backward(torch.ones_like(out_ds), eng._grads, d_ds)
        g_ds = [{k: v.clone() for k, v in g.items()} for g in eng._grads]
    # the same batch through the host-packed path
    eng.set_graph_prepared(ref)
    eng.readout_set_graphs(b.G, nodes_per_graph=b.nodes_per_graph, node_mask=pk["node_mask"])
    h0_ref = torch.from_numpy(pk["initial_node_representation"].reshape(-1, D)).cuda()
    out_ref = eng.forward(h0_ref)
    assert torch.equal(out_ds, out_ref)
    assert torch.equal(ro_ds, _readout(eng, out_ref, h0_ref, seed))
    if save:   # deterministic mode: d h0 and every weight gradient bit for bit
        d_ref = torch.zeros_like(h0_ref)
        for g in eng._grads:
            for v in g.values():
                v.zero_()
        eng.backward(torch.ones_like(out_ref), eng._grads, d_ref)
        assert torch.equal(d_ds, d_ref)
        for a, c in zip(g_ds, eng._grads):
            for k in a:
                assert torch.equal(a[k], c[k]), k


CASES = [  # hidden, precision, tie
    (100, "bf16x3", True), (256, "bf16x3", True), (100, "fp32", True), (100, "bf16x3", False), (24, "bf16", True)]


@pytest.mark.parametrize("hidden,precision,tie", CASES)
@pytest.mark.parametrize("save", [False, True])
def test_dense_dataset_batches_match_the_host_packed_path(hidden, precision, tie, save):
    import torch
    mols = molecules()
    T, p = edge_types(tie), params(hidden)
    eng = PropagationEngine(p, T, precision=precision)
    w = _weights(p, T, hidden)
    eng.set_weights(w)
    eng.set_save_for_backward(save)
    eng.set_deterministic(True)
    eng._grads = [{k: torch.zeros_like(v) for k, v in l.items()} for l in w]
    ds = DeviceDataset.for_engine(eng, flat_of(mols, tie), for_training=save)
    for i, (ids, v) in enumerate(_sequence(mols)):
        b = ds.prepare_batch(ids, save_for_backward=save, nodes_per_graph=v)
        pk = packed(mols, ids, v, hidden, tie)
        # the reference is built in plain host memory: a fresh one is zero in the alignment gaps, as the device image is
        ref = PreparedGraph.host_only_dense(p, T, pk["adjacency_matrix"], precision=precision, num_sms=_sms(), save_for_backward=save)
        _check(eng, b, pk, ref, save, i)
    eng.sync_check()


def test_dense_and_sparse_batches_refuse_the_other_call():
    from tests.test_device_data_cpu import GRU, T as ST, sparse_graph_set
    import torch
    mols = molecules()
    p = params(100)
    eng = PropagationEngine(p, edge_types(True), precision="bf16x3")
    eng.set_weights(_weights(p, edge_types(True), 1))
    ds = DeviceDataset.for_engine(eng, flat_of(mols, True), for_training=False)
    b = ds.prepare_batch([0, 1], save_for_backward=False, nodes_per_graph=29)
    buf = torch.zeros(4 * 29 * 100, device="cuda")
    assert eng.lib.ggnn_set_graph_dataset(eng._h, b._h, buf.data_ptr(), buf.data_ptr(), buf.data_ptr(), eng._stream()) == -1   # GGNN_EINVAL
    assert "ggnn_set_graph_dataset_dense" in eng.lib.ggnn_last_error(eng._h).decode()
    seng = PropagationEngine(dict(GRU, hidden_size=100), ST, precision="bf16x3")
    sds = DeviceDataset.for_engine(seng, packing.FlatSparseGraphs(sparse_graph_set(8), ST), for_training=False)
    sb = sds.prepare_batch([0, 1], save_for_backward=False)
    assert seng.lib.ggnn_set_graph_dataset_dense(seng._h, sb._h, buf.data_ptr(), buf.data_ptr(), buf.data_ptr(), buf.data_ptr(),
                                                 seng._stream()) == -1
    assert "needs a dense dataset batch" in seng.lib.ggnn_last_error(seng._h).decode()
    # and a dense dataset made for one engine shape is refused by another
    other = PropagationEngine(params(64), edge_types(True), precision="bf16x3")
    with pytest.raises(GgnnError, match="different engine configuration"):
        other.set_graph_from_dataset(b)
    eng.sync_check()
    seng.sync_check()
