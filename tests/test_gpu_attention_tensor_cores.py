"""GPU: propagation attention on the streaming wgmma kernels (GGNN_ATT_TENSOR_CORES), forward and every gradient against float64.

The batches, score regimes and helpers are tests/test_attention_edges_cpu.py's and tests/test_gpu_attention_edges.py's.  Each case runs a
forward with save_for_backward and ``ggnn_backward`` on an engine created with ``attention_tensor_cores=True`` and compares the forward
with float64 and ``d h0`` and every weight gradient of every layer, ``edge_type_attention_weights`` included, with float64 autograd of
``oracle.sparse_propagation_torch``.  Bars, max|err| / max|ref| per tensor: bf16x3 1e-4 forward and 2e-4 gradients, bf16 2e-2 (the bars
of tests/test_gpu_weighted_stream.py and tests/test_gpu_wide_hidden.py).

The large / negative score regimes get a bar of their own, derived and not tuned: the scores are taken from the fp32 master of the state,
which after the first step carries the bf16x3 error of the step's GEMMs, eps ~ 2^-16 relative per product (include/ggnn_b200.h).  A score
s = a_t <h[src], h[v]> then carries |s| * 2 eps (two factors), and a softmax probability the same relative error; through the weighted
gather every later quantity inherits it.  With |s| <= S (the largest |step-0 score| of the batch, measured in float64 below) the bar is
2 * (2 S eps), the factor 2 for the gradient's second use of the probabilities, floored at the bf16x3 bars.
"""
import functools

import numpy as np
import pytest

from tests.test_attention_edges_cpu import att_model, batch, regime_h0, regime_weights, step0_scores
from tests.test_gpu_attention_edges import REN, _compare, _rel, _set_env
from tests.test_gpu_backward import _autograd_reference

pytestmark = pytest.mark.gpu

BARS = {"bf16x3": (1e-4, 2e-4), "bf16": (2e-2, 2e-2)}
EPS_BF16X3 = 2.0 ** -16
STREAM_ATT = r"^wgmma-%s STREAM\+attention\(4 launches per step"
DROP_SEED = 4321


def wide_bar(h0, adj, a):
    sc, _ = step0_scores(h0, adj, a)
    return max(BARS["bf16x3"][1], 2.0 * 2.0 * float(np.max(np.abs(sc))) * EPS_BF16X3)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


class Run:
    """One tensor-core attention engine with its weights bound and save_for_backward on."""

    def __init__(self, params, T, w, precision="bf16x3", bwd_precision=None, det=False, keep=1.0):
        from gated_graph_neural_network_samples_b200.engine import PropagationEngine
        self.eng = PropagationEngine(params, T, precision=precision, attention_tensor_cores=True)
        self.rnn_keys = "rnn_kernel" in w[0]   # the oracle's names of the RNN cell's weights
        self.dev_w = [{REN.get(k, k): _cuda(v) for k, v in lw.items()} for lw in w]
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(True)
        if bwd_precision:
            self.eng.set_backward_precision(bwd_precision)
        self.eng.set_deterministic(det)
        if keep < 1.0:
            self.eng.set_state_dropout(keep, DROP_SEED)

    def forward(self, h0):
        self.th0 = _cuda(h0)
        self.out = self.eng.forward(self.th0)   # held: the backward reads h0 and h_out again (the RNN cell's derivative from its output)
        self.eng.sync_check()
        return self.out.cpu().numpy()

    def backward(self, g, fields=None):
        import torch
        grads = [{k: torch.zeros_like(v) for k, v in lw.items() if fields is None or k in fields} for lw in self.dev_w]
        dh0 = torch.zeros_like(self.th0)
        self.eng.backward(_cuda(g), grads, dh0)
        self.eng.sync_check()
        inv = {v: k for k, v in REN.items()}
        return dh0.cpu().numpy(), [{inv.get(k, k) if self.rnn_keys else k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]


def check(name, params, kind, regime="mild", precision="bf16x3", bwd_precision=None, keep=1.0, det=False):
    adj, indeg, T = batch(kind)
    D = params["hidden_size"]
    h0 = regime_h0(regime, indeg.shape[0], D)
    w = regime_weights(params, T, regime)
    g = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    drop = (keep, DROP_SEED) if keep < 1.0 else None
    ref = _autograd_reference(params, T, w, adj, indeg, h0, g, state_dropout=drop)
    r = Run(params, T, w, precision, bwd_precision, det, keep)
    r.eng.set_graph_sparse(adj, indeg)
    assert r.eng.plan.startswith("wgmma-%s STREAM+attention(" % precision), r.eng.plan
    out = r.forward(h0)
    dh0, gw = r.backward(g)
    bar_f, bar_g = BARS[precision]
    if regime in ("large", "negative"):
        bar_f = bar_g = wide_bar(h0, adj, w[0]["edge_type_attention_weights"])
    _compare("tensor-core attention", name, (out, dh0, gw), ref, bar_f, bar_g)
    return adj, gw


WIDTHS = (4, 20, 36, 52, 68, 84, 100, 116, 128, 260, 276, 316, 384, 512)


@pytest.mark.parametrize("D", WIDTHS)
def test_every_width_class(D, monkeypatch):
    _set_env(monkeypatch, {})
    check("width-D%d" % D, att_model(D), "hubs")


@pytest.mark.parametrize("D", [36, 260])
def test_single_bf16_mma(D, monkeypatch):
    _set_env(monkeypatch, {})
    check("bf16-D%d" % D, att_model(D), "hubs", precision="bf16")


@pytest.mark.parametrize("D", [36, 256])
@pytest.mark.parametrize("kind", ["hubs", "big_hub", "self_dup", "t16_all", "t16_ends", "t1"])
def test_degree_and_topology(kind, D, monkeypatch):
    """In-degrees 1 .. 300 and 1100, self-loops and duplicates, 16 types (all / only 0 and 15: absent types get d a_t exactly 0), one type."""
    _set_env(monkeypatch, {})
    adj, gw = check("%s-D%d" % (kind, D), att_model(D), kind)
    absent = [t for t, a in enumerate(adj) if a.shape[0] == 0]
    for lw in gw:
        assert np.all(lw["edge_type_attention_weights"][absent] == 0.0), lw["edge_type_attention_weights"]


@pytest.mark.parametrize("D", [36, 256])
@pytest.mark.parametrize("regime", ["large", "negative", "a_zero", "a_negative"])
def test_score_regimes(regime, D, monkeypatch):
    _set_env(monkeypatch, {})
    check("%s-D%d" % (regime, D), att_model(D), "hubs", regime)


VARIANTS = {
    "rnn": lambda D: att_model(D, cell="RNN"),
    "sum-nobias": lambda D: att_model(D, bias=False, avg=False),
    "zero-step": lambda D: att_model(D, layer_timesteps=(2, 0, 1), residual_connections={"2": [1, 2]}),
    "res4": lambda D: att_model(D, layer_timesteps=(1, 1, 1, 2), residual_connections={"3": [0, 1, 2, 3]}),
}


@pytest.mark.parametrize("D", [36, 260])
@pytest.mark.parametrize("variant", sorted(VARIANTS) + ["dropout"])
def test_model_variants(variant, D, monkeypatch):
    _set_env(monkeypatch, {})
    if variant == "dropout":
        check("dropout-D%d" % D, att_model(D), "hubs", keep=0.8)
    else:
        check("%s-D%d" % (variant, D), VARIANTS[variant](D), "hubs")


@pytest.mark.parametrize("D", [36, 260])
def test_tensor_core_backward_and_deterministic_mode(D, monkeypatch):
    _set_env(monkeypatch, {})
    check("bwd-bf16x3-D%d" % D, att_model(D), "self_dup", bwd_precision="bf16x3")
    check("det-D%d" % D, att_model(D), "self_dup", det=True)


@functools.lru_cache(maxsize=None)
def _inputs(kind, D):
    adj, indeg, T = batch(kind)
    params = att_model(D)
    return params, adj, indeg, T, regime_h0("mild", indeg.shape[0], D), regime_weights(params, T, "mild"), \
        np.random.default_rng(5).normal(size=(indeg.shape[0], D)).astype(np.float32)


@pytest.mark.parametrize("D", [36, 260])
def test_partial_requests_repeats_and_launch_count(D, monkeypatch):
    """Only d a_t and everything but it against a full request; the forward and d h0 bit-identical across repeats and in deterministic
    mode; 1 + steps x (4 GRU / 3 RNN) launches per forward."""
    _set_env(monkeypatch, {})
    params, adj, indeg, T, h0, w, g = _inputs("hubs", D)
    for det in (False, True):
        r = Run(params, T, w, det=det)
        r.eng.set_graph_sparse(adj, indeg)
        out_a = r.forward(h0)
        dh0_a, full = r.backward(g)
        out_b = r.forward(h0)
        assert r.eng.last_launch_count == 1 + 3 * 4
        dh0_b, _ = r.backward(g)
        np.testing.assert_array_equal(out_a, out_b)
        np.testing.assert_array_equal(dh0_a, dh0_b)
        att = ["edge_type_attention_weights"]
        for request in (att, [k for k in r.dev_w[0] if k not in att]):
            dh0, part = r.backward(g, request)
            np.testing.assert_array_equal(dh0, dh0_a)
            for p, f in zip(part, full):
                assert sorted(p) == sorted(request)
                for k in p:
                    assert _rel(p[k], f[k]) < 1e-5, k
    rnn = att_model(D, cell="RNN")
    w = regime_weights(rnn, T, "mild")
    r = Run(rnn, T, w)
    r.eng.set_graph_sparse(adj, indeg)
    r.forward(h0)
    r.forward(h0)
    assert r.eng.last_launch_count == 1 + 3 * 3


@pytest.mark.parametrize("D", [36, 260])
def test_feeds_agree(D, monkeypatch):
    """set_graph_sparse, a prepared graph and a device-dataset batch of the same graphs: identical images, bit-identical final states."""
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset
    from tests.test_device_data_cpu import packed_graph, sparse_graph_set
    _set_env(monkeypatch, {})
    T = 4
    flat = packing.FlatSparseGraphs(sparse_graph_set(), T)
    ids = np.array([5, 2, 9, 0, 31, 17, 40, 3], np.int64)
    pk = packed_graph(flat, ids, D)
    adj, indeg = pk["adjacency_lists"], pk["num_incoming_edges_per_type"]
    params = att_model(D)
    w = regime_weights(params, T, "mild")
    r = Run(params, T, w)
    ds = DeviceDataset.for_engine(r.eng, flat, for_training=True)
    b = ds.prepare_batch(ids, save_for_backward=True)
    h0, _, _ = r.eng.set_graph_from_dataset(b)
    img_ds = r.eng.graph_image()
    out_ds = r.forward(h0.cpu().numpy())
    r.eng.set_graph_sparse(adj, indeg)
    img_sp = r.eng.graph_image()
    out_sp = r.forward(h0.cpu().numpy())
    g = r.eng.prepare_graph_sparse(adj, indeg)
    r.eng.set_graph_prepared(g)
    out_pg = r.forward(h0.cpu().numpy())
    assert "STREAM+attention" in r.eng.plan
    assert img_ds.shape == img_sp.shape and np.array_equal(img_ds, img_sp), np.flatnonzero(img_ds != img_sp)[:32]
    np.testing.assert_array_equal(g.image(), img_sp)
    np.testing.assert_array_equal(out_ds, out_sp)
    np.testing.assert_array_equal(out_pg, out_sp)


def test_poisoned_components_do_not_reach_clean_ones(monkeypatch):
    """The memory canary of tests/test_gpu_canaries.py on the new plan: NaN components leave every clean row's bits alone."""
    import tests.test_gpu_canaries as C
    from tests import test_canaries_cpu as K
    from tests.test_backward_plans_cpu import sparse_batch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    monkeypatch.setattr(C, "PropagationEngine", functools.partial(PropagationEngine, attention_tensor_cores=True))
    _set_env(monkeypatch, {})
    for D in (36, 260):
        c = K.Case("stream-attention-D%d" % D, att_model(D, layer_timesteps=(2, 1)), 4, "mol24", "bf16x3", {}, STREAM_ATT % "bf16x3")
        adj, indeg, h0 = sparse_batch(c.batch, D, c.T)
        w = regime_weights(c.params, c.T, "mild")
        g = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
        r = C.Ggnn(c.params, c.T, w, c.precision, (adj, indeg))
        assert "STREAM+attention" in r.eng.plan, r.eng.plan
        labels, bad_ids = K.sparse_isolation_batch(c, r.eng.prepare_graph_sparse(adj, indeg).arrays(c.T)["tile_start"])[3:]

        def cmp(got, ref, tag):
            err = _rel(got, ref)
            assert err < BARS["bf16x3"][1], (tag, err)
        C._isolation(c.name, r, np.isin(labels, bad_ids), h0, g, C._ggnn_reference(c.params, c.T, w, adj, indeg, 1.0), cmp)


# ---------------------------------------------------------------------------------------------------------------- through the plug-in
@pytest.mark.parametrize("name", ["attention_bias_avg", "attention_rnn_sum"])
def test_reference_fixtures_through_the_plugin(tmp_path, golden_dir, monkeypatch, name):
    """The reference graph code's attention fixtures through SparseGGNNChemModel with --attention-tensor-cores at bf16x3: the loss within
    1e-4 of the fixture, every trainable's gradient within 2e-4 of float64."""
    import tests.test_gpu_chem_ggnn_gradients as G
    plain = G._sparse_model
    monkeypatch.setattr(G, "_sparse_model", lambda tmp, precision, mols, **cfg: _with_option(plain, tmp, precision, mols, **cfg))
    m, z, feed = G._sparse_fixture(tmp_path, golden_dir, name, "bf16x3")
    loss = G._check("refgraph %s tensor-core attention" % name, m, feed, monkeypatch, STREAM_ATT % "bf16x3", "bf16x3")
    assert abs(loss - float(z["loss"])) < 1e-4 * abs(float(z["loss"])), (loss, float(z["loss"]))


def _with_option(plain, tmp, precision, mols, **cfg):
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    return SparseGGNNChemModel({"--log_dir": str(tmp), "--precision": precision, "--train_data": mols[:48], "--valid_data": mols[48:],
                                "--config": cfg, "--attention-tensor-cores": True})


@pytest.mark.parametrize("device_data", [False, True])
def test_plugin_trains_and_predicts(tmp_path, monkeypatch, device_data):
    """A short training run and predict with --attention-tensor-cores, the data on the host or on the device; predict from the other
    feed agrees within the bf16x3 bar, and the engine ran the tensor-core attention plan."""
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    _set_env(monkeypatch, {})
    mols = synthetic.make_molecules(80, seed=4)
    args = {"--log_dir": str(tmp_path), "--precision": "bf16x3", "--train_data": mols[:64], "--valid_data": mols[64:],
            "--attention-tensor-cores": True, "--device-data": device_data,
            "--config": {"hidden_size": 36, "use_propagation_attention": True, "num_epochs": 2, "batch_size": 600,
                         "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}}}
    m = SparseGGNNChemModel(args)
    m.train()
    assert m.engine.plan.startswith("wgmma-bf16x3 STREAM+attention("), m.engine.plan
    pred = np.asarray(m.predict(mols[64:], device_data=device_data))
    again = np.asarray(m.predict(mols[64:], device_data=not device_data))
    assert pred.shape[-1] == 16 and np.all(np.isfinite(pred))
    assert _rel(pred, again) < BARS["bf16x3"][0]
