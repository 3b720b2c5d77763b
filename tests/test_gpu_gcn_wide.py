"""GPU: the sparse GCN's ``wide_hidden`` option -- the streaming wgmma plan above hidden 128 on bf16x3 / bf16 (a weighted gather into the
operand image, then the TMA-fed streaming GEMM with the GCN epilogue) and the fp32 kernel up to 512 -- against the float64 list-order
oracle; the backward pass at 384 and 512 against float64 autograd on both backward precisions; deterministic repeats; the readout;
dataset batches against host-packed ones; refusals of batches prepared with the other flag; guard bands; the plug-in; the benchmark's
100 000-node batch."""
import numpy as np
import pytest

from tests import gcn_oracle as G
from tests._util import max_rel_err

pytestmark = pytest.mark.gpu

BARS = {"bf16x3": 1e-4, "bf16": 2e-2, "fp32": 1e-5}
GRAD_BARS = {"fp32": 2.5e-5, "bf16x3": 2e-4}
SEED = 9091


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def graph(kind, seed=0):
    """(V, list, weights): ``random`` is unsorted, duplicate-bearing and non-symmetric over 300 nodes (V not a multiple of 128) with
    isolated nodes and one row of in-degree 1500; ``small`` has V < 128; ``empty`` has no entries."""
    rng = np.random.default_rng(seed)
    if kind == "empty":
        return 70, np.zeros((0, 2), np.int64), np.zeros(0, np.float32)
    V, nnz = (300, 2000) if kind == "random" else (50, 300)
    lst, w = G.random_gcn_list(V, nnz, rng, isolated=(0, 7, V - 1))
    if kind == "random":   # one very high in-degree row
        hub = np.stack([np.full(1500, 11), rng.integers(1, V - 1, 1500)], 1).astype(np.int64)
        lst = np.concatenate([lst, hub])
        w = np.concatenate([w, rng.uniform(-0.05, 0.05, 1500).astype(np.float32)])
    return V, lst, w


def params(D, L, V, bias, seed):
    rng = np.random.default_rng([D, L, V, seed])
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)] if bias else None
    return rng.normal(0, 1, (V, D)).astype(np.float32), ks, bs


def oracle_states(h0, lst, w, ks, bs=None, masks=None, keep=1.0):
    """Every node_states_per_layer entry in float64, the list-order statement of tests/gcn_oracle.py."""
    L = len(ks)
    out = [np.asarray(h0, np.float64)]
    for l in range(L):
        h = G.gcn_propagation_loops(out[-1], lst, w, [ks[l]], None if bs is None else [bs[l]])
        if l < L - 1:
            h = np.maximum(h, 0.0)
            if masks is not None:
                h = h * masks[l] / np.float64(np.float32(keep))
        out.append(h)
    return out


class Run:
    def __init__(self, D, L, V, lst, w, h0, ks, bs, precision, keep=1.0, save=False, det=False, bwd="fp32"):
        import torch
        from gated_graph_neural_network_samples_b200.engine import GCNEngine
        self.eng = eng = GCNEngine(D, L, use_bias=bs is not None, precision=precision, wide_hidden=True)
        self.dk = [_cuda(k) for k in ks]
        self.db = None if bs is None else [_cuda(b) for b in bs]
        eng.set_weights(self.dk, self.db)
        eng.set_save_for_backward(save)
        eng.set_deterministic(det)
        eng.set_backward_precision(bwd)
        eng.set_graph_gcn(V, lst, w)
        eng.set_state_dropout(keep, SEED)
        self.h0 = _cuda(h0)
        self.L, self.V, self.D = L, V, D
        self.out_t = torch.empty_like(self.h0)
        self.out = self.forward()

    def forward(self):
        self.eng.forward(self.h0, self.out_t)
        self.eng.sync_check()
        return self.out_t.cpu().numpy()

    def backward(self, g_out):
        import torch
        grads = [{"kernel": torch.zeros_like(k), **({"bias": torch.zeros_like(b)} if self.db else {})} for k, b in
                 zip(self.dk, self.db or [None] * self.L)]
        dh0 = torch.full_like(self.h0, np.nan)
        self.eng.backward(_cuda(g_out), grads, d_h0=dh0)
        self.eng.sync_check()
        return dh0.cpu().numpy(), [{k: v.cpu().numpy() for k, v in g.items()} for g in grads]


def _plan_ok(plan, precision):
    return plan.startswith("gcn-fp32-ffma GLOBAL(") if precision == "fp32" else plan.startswith("gcn-stream-%s (" % precision)


# ---------------------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "fp32"])
@pytest.mark.parametrize("D", [132, 256, 260, 384, 512])
def test_forward_and_every_layer_state_match_the_oracle(D, precision):
    L = 4
    V, lst, w = graph("random", D)
    h0, ks, bs = params(D, L, V, True, 1)
    r = Run(D, L, V, lst, w, h0, ks, bs, precision, save=True)
    assert _plan_ok(r.eng.plan, precision), r.eng.plan
    ref = oracle_states(h0, lst, w, ks, bs)
    for l in range(1, L + 1):
        err = max_rel_err(r.eng.layer_state(l).cpu().numpy(), ref[l])
        assert err < BARS[precision], (l, err, r.eng.plan)
    assert max_rel_err(r.out, ref[L]) < BARS[precision]
    if precision != "fp32":
        assert r.eng.last_launch_count >= 2 * L   # a weighted gather and a GEMM per layer (and the weight tiling on the first forward)
    for _ in range(2):   # repeated forwards are bit-identical
        np.testing.assert_array_equal(r.forward(), r.out)


@pytest.mark.parametrize("kind", ["small", "empty"])
@pytest.mark.parametrize("L,bias", [(1, False), (4, True), (2, False)])
def test_small_batches_and_model_shapes(kind, L, bias):
    for D, precision in ((260, "bf16x3"), (384, "bf16")):
        V, lst, w = graph(kind, L)
        h0, ks, bs = params(D, L, V, bias, 2)
        r = Run(D, L, V, lst, w, h0, ks, bs, precision)
        assert _plan_ok(r.eng.plan, precision), r.eng.plan
        ref = oracle_states(h0, lst, w, ks, bs)[-1]
        if kind == "empty":
            np.testing.assert_allclose(r.out, ref, rtol=0, atol=1e-6)
        else:
            assert max_rel_err(r.out, ref) < BARS[precision], (D, precision, max_rel_err(r.out, ref))


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_state_dropout_uses_the_engine_masks(precision):
    D, L, keep = 384, 3, 0.7
    V, lst, w = graph("random", 5)
    h0, ks, bs = params(D, L, V, True, 3)
    r = Run(D, L, V, lst, w, h0, ks, bs, precision, keep=keep, save=True)
    masks = [r.eng.state_dropout_mask(l, keep, SEED) for l in range(L - 1)]
    assert all(0.6 < m.mean() < 0.8 for m in masks)
    ref = oracle_states(h0, lst, w, ks, bs, masks, keep)
    for l in range(1, L + 1):
        assert max_rel_err(r.eng.layer_state(l).cpu().numpy(), ref[l]) < BARS[precision], l
    # dropped units are exactly zero where the mask says so
    for l in range(1, L):
        assert np.all(r.eng.layer_state(l).cpu().numpy()[masks[l - 1] == 0] == 0)


# ---------------------------------------------------------------------------------------------------------------- backward
def _pattern_propagation(th0, lst, w, tk, tb, patterns, keep):
    """The float64 forward with relu and dropout replaced by ``x * patterns[l] / keep`` (the engine's side of every relu kink: ``patterns``
    are its saved layer outputs' ``y > 0``), differentiable in h0 and the weights."""
    import torch
    rows, cols = torch.from_numpy(np.asarray(lst[:, 0], np.int64)), torch.from_numpy(np.asarray(lst[:, 1], np.int64))
    wt, h = torch.from_numpy(w).double(), th0
    for l in range(len(tk)):
        h = torch.zeros_like(h).index_add_(0, rows, wt[:, None] * h[cols]) @ tk[l] + tb[l]
        if l < len(tk) - 1:
            h = h * torch.from_numpy(patterns[l].astype(np.float64)) / float(np.float32(keep))
    return h


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("D", [384, 512])
def test_gradients_match_float64_autograd(D, bwd):
    """dW, db and d h0 against float64 autograd through the engine's relu / dropout pattern; where that pattern and float64's disagree
    (a pre-activation within the forward's rounding of 0), the float64 pre-activation must be that small."""
    import torch
    L, keep = 3, 0.8
    V, lst, w = graph("random", D + 1)
    h0, ks, bs = params(D, L, V, True, 4)
    r = Run(D, L, V, lst, w, h0, ks, bs, "bf16x3", keep=keep, save=True, bwd=bwd)
    states = [r.eng.layer_state(l).cpu().numpy() for l in range(1, L)]
    g_out = np.random.default_rng(6).normal(0, 1, (V, D)).astype(np.float32)
    dh0, grads = r.backward(g_out)
    masks = [r.eng.state_dropout_mask(l, keep, SEED) for l in range(L - 1)]
    patterns = [y > 0 for y in states]
    h = np.asarray(h0, np.float64)
    for l in range(L - 1):   # the kink check, layer by layer on the float64 states
        pre = G.gcn_propagation_loops(h, lst, w, [ks[l]], [bs[l]])
        dis = patterns[l] != ((pre > 0) & (masks[l] > 0))
        assert not dis.any() or np.abs(pre[dis]).max() < BARS["bf16x3"] * np.abs(pre).max(), (l, np.abs(pre[dis]).max())
        h = np.maximum(pre, 0.0) * masks[l] / np.float64(np.float32(keep))
    th0 = torch.from_numpy(h0).double().requires_grad_()
    tk = [torch.from_numpy(k).double().requires_grad_() for k in ks]
    tb = [torch.from_numpy(b).double().requires_grad_() for b in bs]
    _pattern_propagation(th0, lst, w, tk, tb, patterns, keep).backward(torch.from_numpy(g_out).double())
    bar = GRAD_BARS[bwd]
    for l in range(L):
        assert max_rel_err(grads[l]["kernel"], tk[l].grad.numpy()) < bar, (l, "kernel")
        assert max_rel_err(grads[l]["bias"], tb[l].grad.numpy()) < bar, (l, "bias")
    assert max_rel_err(dh0, th0.grad.numpy()) < bar


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
def test_deterministic_mode_repeats_bit_for_bit(bwd):
    D, L = 512, 3
    V, lst, w = graph("random", 8)
    h0, ks, bs = params(D, L, V, True, 5)
    r = Run(D, L, V, lst, w, h0, ks, bs, "bf16x3", keep=0.9, save=True, det=True, bwd=bwd)
    g_out = np.random.default_rng(7).normal(0, 1, (V, D)).astype(np.float32)
    a = r.backward(g_out)
    r2 = Run(D, L, V, lst, w, h0, ks, bs, "bf16x3", keep=0.9, save=True, det=True, bwd=bwd)
    np.testing.assert_array_equal(r2.out, r.out)
    for d0, d1 in ((a, r.backward(g_out)), (a, r2.backward(g_out))):
        np.testing.assert_array_equal(d0[0], d1[0])
        for g0, g1 in zip(d0[1], d1[1]):
            for k in g0:
                np.testing.assert_array_equal(g0[k], g1[k])


def test_readout_at_512():
    import torch
    D, L = 512, 2
    rng = np.random.default_rng(6)
    V, lst, w = G.component_list([40, 100, 70], rng)
    h0, ks, bs = params(D, L, V, False, 6)
    r = Run(D, L, V, lst, w, h0, ks, bs, "bf16x3")
    gnl = np.repeat(np.arange(3, dtype=np.int32), [40, 100, 70])
    r.eng.readout_set_graphs(3, gnl)
    wg, bg, wt, bt = (_cuda(rng.normal(0, 0.05, n)) for n in (2 * D, 1, D, 1))
    hl = r.out_t
    out = r.eng.readout_forward(hl, r.h0, wg, bg, wt, bt).cpu().numpy()
    hl64, hz64 = hl.double(), r.h0.double()
    gate = torch.sigmoid(torch.cat([hl64, hz64], 1) @ wg.double() + bg.double()) * (hl64 @ wt.double() + bt.double())
    ref = torch.zeros(3, dtype=torch.float64, device="cuda").index_add_(0, torch.from_numpy(gnl).long().cuda(), gate).cpu().numpy()
    assert max_rel_err(out, ref) < 1e-5


# ---------------------------------------------------------------------------------------------------------------- datasets, refusals, guard bands
@pytest.mark.parametrize("hidden,precision", [(256, "bf16x3"), (512, "bf16")])
@pytest.mark.parametrize("save", [False, True])
def test_dataset_batches_match_the_feed_dict_path(hidden, precision, save):
    import torch
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GCNEngine, PreparedGraph
    from tests.test_device_data_cpu import gcn_graph_set
    from tests.test_gpu_device_data import _batches, _check_batch, _sms
    flat = packing.FlatGCNGraphs(gcn_graph_set())
    eng = GCNEngine(hidden, 3, use_bias=True, precision=precision, wide_hidden=True)
    g = torch.Generator().manual_seed(hidden)
    ks = [(torch.rand(hidden, hidden, generator=g) * 0.2 - 0.1).cuda() for _ in range(3)]
    bs = [(torch.rand(hidden, generator=g) * 0.2 - 0.1).cuda() for _ in range(3)]
    eng.set_weights(ks, bs)
    eng.set_save_for_backward(save)
    eng.set_deterministic(True)
    eng._grads = [{"kernel": torch.zeros_like(k), "bias": torch.zeros_like(b)} for k, b in zip(ks, bs)]
    ds = DeviceDataset.for_engine(eng, flat, for_training=save)
    for i, ids in enumerate(_batches(flat.num_graphs)[:8]):
        b = ds.prepare_batch(ids, save_for_backward=save)
        packed = flat.pack(ids, hidden) if len(ids) else None
        V, lst, w = ((packed["initial_node_representation"].shape[0], packed["adjacency_list"], packed["adjacency_weights"]) if packed is not None
                     else (0, np.zeros((0, 2), np.int64), np.zeros(0)))
        ref = PreparedGraph.host_only_gcn(hidden, 3, V, lst, w, use_bias=True, precision=precision, num_sms=_sms(), save_for_backward=save,
                                          wide_hidden=True)
        if V:
            assert ref.info()["plan"].startswith("gcn-stream-"), ref.info()["plan"]
        _check_batch(eng, b, packed, ref, save, i)
    eng.sync_check()


@pytest.mark.parametrize("D", [100, 256])
def test_a_batch_prepared_with_the_other_flag_is_refused(D):
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GCNEngine, GgnnError, PreparedGraph
    from tests.test_device_data_cpu import gcn_graph_set
    from tests.test_gpu_device_data import _sms
    V, lst, w = graph("small")
    wide, narrow = (GCNEngine(D, 2, precision="bf16x3", wide_hidden=f) for f in (True, False))
    for eng, other in ((wide, False), (narrow, True)):
        g = PreparedGraph.host_only_gcn(D, 2, V, lst, w, precision="bf16x3", num_sms=_sms(), wide_hidden=other)
        with pytest.raises(GgnnError, match="different engine configuration"):
            eng.set_graph_prepared(g)
    flat = packing.FlatGCNGraphs(gcn_graph_set(6))
    for a, b in ((wide, narrow), (narrow, wide)):
        ds = DeviceDataset.for_engine(a, flat, for_training=False)
        with pytest.raises(GgnnError, match="different engine configuration"):
            b.set_graph_from_dataset(ds.prepare_batch([0, 1], save_for_backward=False))
        a.set_graph_from_dataset(ds.prepare_batch([0, 1], save_for_backward=False))   # its own engine takes it


@pytest.mark.parametrize("D,V", [(260, 129), (512, 65)])
def test_guard_bands_around_every_buffer(D, V):
    import torch
    from tests import test_canaries_cpu as K
    from tests.test_gpu_canaries import _g
    L = 2
    rng = np.random.default_rng(D)
    Vc, lst, w = G.component_list([int(x) for x in np.diff(np.r_[0, np.sort(rng.choice(np.arange(1, V), 4, replace=False)), V])], rng)
    assert Vc == V
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)]
    h0, g = rng.normal(0, 1, (V, D)).astype(np.float32), rng.normal(0, 1, (V, D)).astype(np.float32)
    pk, pb = rng.normal(0, 1, (D, D)).astype(np.float32), rng.normal(0, 1, D).astype(np.float32)

    def run(guard, precision):
        from gated_graph_neural_network_samples_b200.engine import GCNEngine
        keep = []

        def buf(s, f=None):
            if guard:
                b = _g(s, f)
                keep.append(b)
                return b.t
            return (_cuda(f) if f is not None else torch.empty(s, device="cuda")).reshape(s)
        eng = GCNEngine(D, L, use_bias=True, precision=precision, wide_hidden=True)
        eng.set_deterministic(True)
        eng.set_weights([buf((D, D), k) for k in ks], [buf((D,), b) for b in bs])
        eng.set_save_for_backward(True)
        eng.set_graph_gcn(V, lst, w)
        assert _plan_ok(eng.plan, precision), eng.plan
        th0, out = buf((V, D), h0), buf((V, D))
        eng.forward(th0, out)
        grads = [{"kernel": buf((D, D), pk), "bias": buf((D,), pb)} for _ in range(L)]
        dh0 = buf((V, D))
        eng.backward(buf((V, D), g), grads, dh0)
        eng.sync_check()
        outs = [out, dh0] + [t for d in grads for t in d.values()]
        if guard:
            assert not any(K.has_payload(t) for t in outs)
            assert all(b.bands_intact() for b in keep)
        return [t.cpu().numpy() for t in outs]

    for precision in ("bf16x3", "bf16"):
        for a, b in zip(run(True, precision), run(False, precision)):
            np.testing.assert_array_equal(a, b, err_msg=precision)


# ---------------------------------------------------------------------------------------------------------------- plug-in and the benchmark batch
def test_plugin_trains_two_steps_at_hidden_512(tmp_path):
    import torch
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    mols = synthetic.make_molecules(40, seed=3)
    m = SparseGCNChemModel({"--log_dir": str(tmp_path), "--precision": "bf16x3", "--gcn-wide-hidden": True, "--train_data": mols[:30],
                            "--valid_data": mols[30:], "--config": {"hidden_size": 510, "batch_size": 350, "num_timesteps": 3,
                                                                    "learning_rate": 0.001, "num_epochs": 1}})
    assert m.engine.D == 512 and m.engine.wide_hidden
    before = [t.detach().clone() for t in m.weights["edge_weights"]]
    loss, _, _, _, steps = m.run_epoch("train", m.train_data, True)
    assert steps >= 2 and np.isfinite(loss), (steps, loss)
    assert m.engine.plan.startswith("gcn-stream-bf16x3 ("), m.engine.plan
    assert all(not torch.equal(a, b) for a, b in zip(before, m.weights["edge_weights"]))
    assert np.isfinite(m.run_epoch("valid", m.valid_data, False)[0])


def _reference_on_gpu(V, lst, w, h0, ks):
    """float64 on the device (the 100 000-node batch): S = index_add in list order, then S . W, relu between layers."""
    import torch
    rows = torch.from_numpy(np.ascontiguousarray(lst[:, 0])).cuda()
    cols = torch.from_numpy(np.ascontiguousarray(lst[:, 1])).cuda()
    wt = torch.from_numpy(np.asarray(w, np.float64)).cuda()
    h = torch.from_numpy(h0).cuda().double()
    for l, k in enumerate(ks):
        h = torch.zeros_like(h).index_add_(0, rows, wt[:, None] * h[cols]) @ torch.from_numpy(k).cuda().double()
        if l < len(ks) - 1:
            h = torch.relu(h)
    return h.cpu().numpy()


@pytest.mark.parametrize("D", [256, 512])
def test_benchmarked_batch(D):
    from tests.test_gcn_tiles_cpu import batch
    V, lst, w = batch("bench")
    L = 4
    rng = np.random.default_rng(D)
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    ref = _reference_on_gpu(V, lst, w, h0, ks)
    for precision in ("bf16x3", "fp32"):
        r = Run(D, L, V, lst, w, h0, ks, None, precision)
        assert V > 90000 and _plan_ok(r.eng.plan, precision), r.eng.plan   # the plug-in's 100 000-node budget: 99 046 nodes
        err = max_rel_err(r.out, ref)
        print("\nbench D=%d %-6s %.2e  %s" % (D, precision, err, r.eng.plan[:70]))
        assert err < BARS[precision], (precision, err)
