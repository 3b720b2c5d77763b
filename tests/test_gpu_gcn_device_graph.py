"""GPU: sparse GCN batches built on the device from a CUDA adjacency list (``set_graph_gcn_device``, DESIGN 2.16).

The host builder is the oracle: for the same list, the device build must leave the engine with ``prepare_graph_gcn_message_weighted`` +
``set_graph_prepared``'s plan text, message count and graph image, every byte included.  Covered:

1. bytes on every GCN plan of tests/test_gpu_gcn_message_weights.py (the wgmma kernel LOCAL at 12 / 100 / 128 and GLOBAL with a 150-node
   component, bf16 LOCAL, the fp32 kernel at 100 / 132 / 256, bf16x3 at 256 without wide_hidden, the streaming plan at 256 / 384 / 512),
   save_for_backward off and on, on the plan's own batch (unsorted, duplicates, self-loops, isolated trailing nodes), the reference
   packer's molecules, the 100 000-node batch, a one-entry non-symmetric list, nnz = 0 and V = 0; a second device build gives the same
   image;
2. on every plan, the forward, every layer state, d h0, dW, db and d w bit-identical to the host-prepared message-weighted batch with the
   same weights (deterministic mode, both backward precisions), and the forward bit-identical to ``set_graph_gcn`` with host weights --
   the LOCAL kernel's shared-memory plan reads the per-tile maxima, so this is where a wrong maximum would show;
3. refusals with the host builder's code and text, and no batch left behind by a failed call;
4. one engine alternating device-built, host-prepared (weighted and message-weighted) and dataset batches, each equal to a fresh engine's;
5. guard bands around the caller's list;
6. SparseGCNChemModel training steps with a CUDA feed against the host feed, and a requires_grad ``adjacency_weights`` against float64.
"""
import numpy as np
import pytest

from tests import test_gpu_gcn_message_weights as GMW
from tests import test_canaries_cpu as K
from tests._util import max_rel_err

pytestmark = pytest.mark.gpu


def _codes():
    """The GGNN_E* values of the header (read, not assumed)."""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "ggnn_b200.h")) as f:
        return {k: int(v) for k, v in re.findall(r"(GGNN_E[A-Z]+)\s*=\s*(-?\d+)", f.read())}


CODES = _codes()
PLANS = GMW.PLANS


# ---------------------------------------------------------------------------------------------------------------- batches
def packer_batch():
    """The reference packer's feed (packing.pack_gcn_batch) of 80 synthetic molecules: V, [nnz, 2] int64 list, [nnz] weights."""
    from gated_graph_neural_network_samples_b200 import packing, synthetic
    f = packing.pack_gcn_batch(packing.process_raw_graphs_gcn(synthetic.make_molecules(80, seed=11)), 100)
    return f["initial_node_representation"].shape[0], np.asarray(f["adjacency_list"], np.int64), f["adjacency_weights"].astype(np.float32)


def batch(kind, plan=None):
    if kind == "plan":   # the plan's own batch: unsorted, duplicate entries, self-loops, isolated trailing nodes
        return GMW.graph(PLANS[plan][4])
    if kind == "packer":
        return packer_batch()
    if kind == "100k":
        from tests.test_gcn_tiles_cpu import batch as tiles_batch
        V, lst, w = tiles_batch("bench")
        return V, np.asarray(lst, np.int64), w
    if kind == "one":    # one entry, not symmetric
        return 5, np.array([[3, 1]], np.int64), np.array([0.75], np.float32)
    if kind == "nnz0":
        return 7, np.zeros((0, 2), np.int64), np.zeros(0, np.float32)
    if kind == "v0":
        return 0, np.zeros((0, 2), np.int64), np.zeros(0, np.float32)
    raise KeyError(kind)


def _cuda_list(lst):
    import torch
    return torch.from_numpy(np.ascontiguousarray(lst, np.int64).reshape(-1, 2)).cuda()


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def gcn_engine(name, L=3, bias=True):
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    D, precision, wide, _, _, _ = PLANS[name]
    return GCNEngine(D, L, use_bias=bias, precision=precision, wide_hidden=wide)


def assert_same_image(got, want, tag):
    assert got.nbytes == want.nbytes, (tag, got.nbytes, want.nbytes)
    if not np.array_equal(got, want):
        diff = np.nonzero(got != want)[0]
        pytest.fail("%s: %d bytes differ, first at %d (device %d, host %d)" % (tag, diff.size, diff[0], got[diff[0]], want[diff[0]]))


# ---------------------------------------------------------------------------------------------------------------- 1. bytes
BATCHES = ["plan", "packer", "100k", "one", "nnz0", "v0"]


@pytest.mark.parametrize("kind", BATCHES)
@pytest.mark.parametrize("name", sorted(PLANS))
def test_device_image_equals_host_image(name, kind):
    import re
    V, lst, _ = batch(kind, name)
    eng = gcn_engine(name)
    for save in (False, True):
        eng.set_save_for_backward(save)
        g = eng.prepare_graph_gcn_message_weighted(V, lst)
        info = g.info()
        dl = _cuda_list(lst)
        eng.set_graph_gcn_device(V, dl)
        tag = "%s %s save=%s" % (name, kind, save)
        assert eng.plan == info["plan"], (tag, eng.plan, info["plan"])
        assert eng.plan.endswith(GMW.TAG), eng.plan
        if kind == "plan":
            assert re.search(PLANS[name][5], eng.plan), (tag, eng.plan)
        assert eng.num_messages() == info["num_messages"] == lst.shape[0]
        got = eng.graph_image()
        assert_same_image(got, g.image(), tag)
        eng.set_graph_gcn_device(V, dl)   # a second build of the same list
        assert_same_image(eng.graph_image(), got, tag + " rebuild")


# ---------------------------------------------------------------------------------------------------------------- 2. bits through the kernels
def add_device_built(r, name, det=True, bwd="fp32"):
    """A third engine on Run r's batch and weights, its graph built on the device (r.engines["built"])."""
    import torch
    eng = gcn_engine(name, r.L, r.bs is not None)
    eng.set_weights(r.dk, r.db)
    eng.set_save_for_backward(True)
    eng.set_deterministic(det)
    eng.set_backward_precision(bwd)
    eng.set_state_dropout(r.keep, GMW.SEED)
    eng.set_graph_gcn_device(r.V, _cuda_list(r.lst))
    assert eng.plan == r.dev.plan, (eng.plan, r.dev.plan)
    eng.set_message_weights(_cuda(r.w))
    r.engines["built"] = eng
    r.outs["built"] = torch.empty_like(r.th0)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("bwd", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", sorted(PLANS))
def test_forward_and_gradients_bit_identical_to_host_batches(name, bwd):
    r = GMW.Run(name, bwd=bwd, det=True)
    add_device_built(r, name, det=True, bwd=bwd)
    built, prepared, host = r.forward("built"), r.forward("dev"), r.forward("host")
    assert np.all(np.isfinite(built))
    np.testing.assert_array_equal(_bits(built), _bits(prepared))
    np.testing.assert_array_equal(_bits(built), _bits(host))   # the host-weighted set_graph_gcn batch
    for l, (a, b) in enumerate(zip(r.states("built"), r.states("dev"))):
        np.testing.assert_array_equal(_bits(a), _bits(b), err_msg="layer %d" % (l + 1))
    g_out = GMW._g_out(r.V, r.D)
    dw, dh0, gw = r.backward(g_out, "built")
    pdw, pdh0, pgw = r.backward(g_out, "dev")
    np.testing.assert_array_equal(_bits(dw), _bits(pdw))
    np.testing.assert_array_equal(_bits(dh0), _bits(pdh0))
    for l in range(r.L):
        assert sorted(gw[l]) == sorted(pgw[l])
        for k in gw[l]:
            np.testing.assert_array_equal(_bits(gw[l][k]), _bits(pgw[l][k]), err_msg="layer %d %s" % (l, k))


# ---------------------------------------------------------------------------------------------------------------- 3. refusals
def _host_error(eng, V, lst):
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    with pytest.raises(GgnnError) as h:
        eng.prepare_graph_gcn_message_weighted(V, lst)
    return h.value


def _device_error(eng, V, lst):
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    with pytest.raises(GgnnError) as d:
        eng.set_graph_gcn_device(V, _cuda_list(lst))
    return d.value


def _assert_no_batch(eng, V, D):
    import torch
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    with pytest.raises(GgnnError) as f:
        eng.forward(torch.zeros(max(V, 1), D, device="cuda"))
    assert f.value.code == CODES["GGNN_ESTATE"]


BAD = {
    "negative": [(1000, 1, -1)],
    "equal-V": [(2000, 0, "V")],
    "above-2^31": [(3000, 1, 2 ** 31 + 7)],
    "wraps-into-range": [(4000, 0, 2 ** 32 + 1)],    # an int32 cast would read node 1
    # list order, not thread order: in the 100 000-node batch a grid-stride thread with a low id reaches entries far down the list on its
    # later iterations, after higher ids have seen earlier ones; the named entry is the first in list order whatever lands first
    "several": [(270341, 0, -5), (20000, 1, "V"), (270400, 1, 2 ** 40), ("last", 0, -1)],
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_first_bad_entry_named_like_the_host_builder(case):
    V, lst, _ = batch("100k")
    lst = lst.copy()
    first = None
    for k, col, val in BAD[case]:
        k = lst.shape[0] - 1 if k == "last" else k
        lst[k, col] = V if val == "V" else val
        first = k if first is None else min(first, k)
    eng = gcn_engine("local-100")
    good = batch("100k")[1]
    eng.set_graph_gcn_device(V, _cuda_list(good))   # a good batch, which the refused call forgets
    host = _host_error(eng, V, lst)
    got = _device_error(eng, V, lst)
    assert got.code == CODES["GGNN_ERANGE"]
    assert str(got) == str(host), (str(got), str(host))
    assert "adjacency_list[%d] = (%d, %d)" % (first, lst[first, 0], lst[first, 1]) in str(got)
    _assert_no_batch(eng, V, 100)


def test_library_refusals():
    import ctypes as C
    import torch
    from gated_graph_neural_network_samples_b200.engine import GgnnError, PropagationEngine
    V, lst, w = batch("packer")
    eng = gcn_engine("local-100")
    lib, h, st = eng.lib, eng._h, eng._stream()
    dl = _cuda_list(lst)
    eng.set_graph_gcn_device(V, dl)
    # host memory behind the Python checks
    host = np.ascontiguousarray(lst)
    assert lib.ggnn_set_graph_gcn_device(h, V, host.shape[0], host.ctypes.data, st) == CODES["GGNN_EINVAL"]
    _assert_no_batch(eng, V, 100)
    # null / negative arguments
    assert lib.ggnn_set_graph_gcn_device(h, V, 4, None, st) == CODES["GGNN_EINVAL"]
    assert lib.ggnn_set_graph_gcn_device(h, -1, 0, None, st) == CODES["GGNN_EINVAL"]
    assert lib.ggnn_set_graph_gcn_device(h, V, -1, dl.data_ptr(), st) == CODES["GGNN_EINVAL"]
    # more entries than int32 indexing holds, refused before any of them is read: a small valid pointer
    small = _cuda_list(np.zeros((1, 2), np.int64))
    assert lib.ggnn_set_graph_gcn_device(h, V, 2 ** 31, small.data_ptr(), st) == CODES["GGNN_EUNSUPPORTED"]
    _assert_no_batch(eng, V, 100)
    # a GGNN engine refuses the call (and a GCN engine the GGNN one)
    ggnn = PropagationEngine({"hidden_size": 32, "layer_timesteps": [1], "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}, 1,
                             precision="bf16x3")
    assert ggnn.lib.ggnn_set_graph_gcn_device(ggnn._h, V, lst.shape[0], dl.data_ptr(), ggnn._stream()) == CODES["GGNN_ESTATE"]
    assert "GCN call" in ggnn.lib.ggnn_last_error(ggnn._h).decode()
    counts = (C.c_int32 * 1)(lst.shape[0])
    ptrs = (C.c_void_p * 1)(dl.data_ptr())
    assert lib.ggnn_set_graph_sparse_device(h, V, ptrs, counts, None, 0, st) == CODES["GGNN_ESTATE"]
    # a forward before the weights
    eng.set_weights([_cuda(k) for k in GMW.weights(100, 3, True, 0)[0]], [_cuda(b) for b in GMW.weights(100, 3, True, 0)[1]])
    eng.set_graph_gcn_device(V, dl)
    with pytest.raises(GgnnError) as f:
        eng.forward(torch.zeros(V, 100, device="cuda"))
    assert f.value.code == CODES["GGNN_ESTATE"]
    eng.set_message_weights(_cuda(w))
    out = eng.forward(torch.zeros(V, 100, device="cuda"))
    eng.sync_check()
    assert out.shape == (V, 100)


# ---------------------------------------------------------------------------------------------------------------- 4. lifecycle
def _fresh_and_reused(name, steps):
    """Runs every step on one engine and on a fresh engine each; returns the pairs of outputs."""
    import torch
    ks, bs = GMW.weights(PLANS[name][0], 3, True, 5)
    dk, db = [_cuda(k) for k in ks], [_cuda(b) for b in bs]

    def new():
        e = gcn_engine(name)
        e.set_weights(dk, db)
        e.set_deterministic(True)
        e.set_save_for_backward(False)
        return e

    shared, pairs = new(), []
    for step in steps:
        outs = []
        for eng in (shared, new()):
            h0 = step(eng)
            outs.append(eng.forward(h0).cpu().numpy())
            eng.sync_check()
        pairs.append(outs)
    return pairs


def test_one_engine_alternates_device_host_and_dataset_batches():
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset
    from tests.test_device_data_cpu import gcn_graph_set
    name = "local-100"
    D = PLANS[name][0]
    flat = packing.FlatGCNGraphs(gcn_graph_set())
    rng = np.random.default_rng(3)

    def h0_for(V):
        return _cuda(rng.normal(0, 1, (V, D)))

    def device(kind, seed):
        V, lst, w = GMW.graph(kind, seed)
        h0 = h0_for(V)

        def step(eng):
            eng.set_graph_gcn_device(V, _cuda_list(lst))
            eng.set_message_weights(_cuda(w))
            return h0
        return step

    def host(kind, seed, message_weighted):
        V, lst, w = GMW.graph(kind, seed)
        h0 = h0_for(V)

        def step(eng):
            if message_weighted:
                eng.set_graph_prepared(eng.prepare_graph_gcn_message_weighted(V, lst))
                eng.set_message_weights(_cuda(w))
            else:
                eng.set_graph_prepared(eng.prepare_graph_gcn(V, lst, w))
            return h0
        return step

    def dataset(ids):
        def step(eng):
            if not hasattr(eng, "test_dataset"):   # one upload per engine, kept with it
                eng.test_dataset = DeviceDataset.for_engine(eng, flat, for_training=False)
            b = eng.test_dataset.prepare_batch(ids, save_for_backward=False)
            h0, _, _ = eng.set_graph_from_dataset(b)
            eng.test_batch = b   # alive until the engine's next upload
            return h0
        return step

    ids = np.arange(flat.num_graphs)
    steps = [device("mol", 1), host("mol", 2, False), dataset(ids[::3]), device("big", 3), host("big", 4, True), device("mol", 5),
             dataset(ids[1::2]), host("mol", 6, True), device("mol", 7)]
    for k, (a, b) in enumerate(_fresh_and_reused(name, steps)):
        assert np.all(np.isfinite(a)), k
        np.testing.assert_array_equal(_bits(a), _bits(b), err_msg="step %d" % k)


# ---------------------------------------------------------------------------------------------------------------- 5. canaries
@pytest.mark.parametrize("name,kind", [("local-100", "packer"), ("stream-384", "plan"), ("fp32-132", "plan")])
def test_guard_bands_around_the_list_stay_unread(name, kind):
    """The list sits between two bands of payload words, which as int64 entries are far out of range (0x7fc0dead7fc0dead).  A read of a
    band would be refused: the call succeeds, the image is the host builder's and the bands are untouched."""
    import torch
    V, lst, _ = batch(kind, name)
    eng = gcn_engine(name)
    eng.set_save_for_backward(True)
    want = eng.prepare_graph_gcn_message_weighted(V, lst).image()
    g = K.guarded(2 * lst.size)   # int64 entries are two words each
    ints = g.view.view(torch.int64)
    ints[:lst.size].copy_(_cuda_list(lst).reshape(-1))
    eng.set_graph_gcn_device(V, ints[:lst.size].reshape(-1, 2))
    assert_same_image(eng.graph_image(), want, "guarded %s %s" % (name, kind))
    assert g.bands_intact()


# ---------------------------------------------------------------------------------------------------------------- 6. the plug-in
def _model(tmp_path, precision, hidden):
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    mols = synthetic.make_molecules(64, seed=5)
    return SparseGCNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:48], "--valid_data": mols[48:],
                               "--config": dict(hidden_size=hidden, num_timesteps=3, gcn_use_bias=True, batch_size=400, random_seed=3)})


def _feed(m):
    feed = dict(next(iter(m.make_minibatch_iterator(m.train_data, True))))
    feed.pop("_prepared_graph", None)
    feed[m.placeholders["graph_state_keep_prob"]] = 1.0
    return feed


def _to_cuda(feed, m):
    import torch
    f = dict(feed)
    f[m.placeholders["adjacency_list"]] = torch.from_numpy(np.asarray(feed[m.placeholders["adjacency_list"]], np.int64)).cuda()
    f[m.placeholders["adjacency_weights"]] = torch.from_numpy(np.asarray(feed[m.placeholders["adjacency_weights"]], np.float32)).cuda()
    return f


@pytest.mark.parametrize("precision,hidden", [("fp32", 32), ("bf16x3", 32), ("bf16x3", 30)])
def test_plugin_training_steps_with_a_cuda_feed(tmp_path, precision, hidden):
    """Three SparseGCNChemModel training steps in deterministic mode from the same start: the CUDA feed gives the host feed's losses,
    gradients and checkpoint, bit for bit (hidden 30 runs zero-padded to 32)."""
    import torch
    results = []
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)   # the engine's fixed-order sums; torch's own ops only warn
    try:
        for device in (False, True):
            torch.manual_seed(0)
            m = _model(tmp_path / ("dev" if device else "host"), precision, hidden)
            m.make_train_step()
            feed = _feed(m)
            f = _to_cuda(feed, m) if device else feed
            variables = [v for _, v in m.graph_model_variables()]
            losses, grads = [], []
            for _ in range(3):
                loss = m.forward_batch(f)[0]
                gs = torch.autograd.grad(loss, variables)
                losses.append(float(loss.detach()))
                grads.append([g.cpu().numpy() for g in gs])
                with torch.no_grad():   # a plain SGD step, so that later steps see other weights
                    for v, g in zip(variables, gs):
                        v -= 0.01 * g
            path = str(tmp_path / ("ckpt-dev.pickle" if device else "ckpt-host.pickle"))
            m.save_progress(path, 3, 0)
            results.append((losses, grads, m.engine.plan, path))
    finally:
        torch.use_deterministic_algorithms(was)
    (lh, gh, ph, ch), (ld, gd, pd, cd) = results
    assert pd == ph + GMW.TAG and ld == lh, (pd, ph, ld, lh)
    for a, b in zip(gd, gh):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(_bits(x), _bits(y))
    import pickle
    with open(ch, "rb") as f1, open(cd, "rb") as f2:
        host_ckpt, dev_ckpt = pickle.load(f1), pickle.load(f2)
    hw, dw = host_ckpt["weights"], dev_ckpt["weights"]
    assert sorted(hw) == sorted(dw)
    for k in hw:
        np.testing.assert_array_equal(np.asarray(hw[k]), np.asarray(dw[k]), err_msg=k)


def test_plugin_adjacency_weights_receive_their_gradient(tmp_path):
    """A requires_grad CUDA adjacency_weights in the feed gets d w, against float64 autograd of the same propagation."""
    import torch
    m = _model(tmp_path, "bf16x3", 32)   # (the engine's default fp32 backward)
    feed = _to_cuda(_feed(m), m)
    w = feed[m.placeholders["adjacency_weights"]].clone().requires_grad_(True)
    feed[m.placeholders["adjacency_weights"]] = w
    m.feed = feed
    with torch.enable_grad():
        h = m.compute_final_node_representations()
    L = m.params["num_timesteps"]
    relu_on = [m.engine.layer_state(l).cpu().numpy() > 0 for l in range(1, L)]   # the engine's relu pattern, as tests/gcn_oracle's checks use
    g_out = torch.from_numpy(np.random.default_rng(2).normal(0, 1, tuple(h.shape)).astype(np.float32)).cuda()
    (dw,) = torch.autograd.grad(h, [w], g_out)
    lst = feed[m.placeholders["adjacency_list"]]
    rows, cols = lst[:, 0], lst[:, 1]
    h0 = m.initial_node_representation_tensor().detach().double()
    w64 = w.detach().double().requires_grad_(True)
    x = h0
    for l in range(L):
        x = torch.zeros_like(x).index_add_(0, rows, w64[:, None] * x[cols]) @ m.weights["edge_weights"][l].detach().double()
        x = x + m.weights["edge_biases"][l].detach().double()
        if l < L - 1:
            x = x * torch.from_numpy(relu_on[l]).cuda().double()
    (rdw,) = torch.autograd.grad(x, [w64], g_out.double())
    err = max_rel_err(dw.cpu().numpy(), rdw.cpu().numpy())
    print("\nGCNDEV plug-in d w %.2e" % err)
    assert err < 2.5e-5, err
