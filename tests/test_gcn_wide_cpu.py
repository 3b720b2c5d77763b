"""CPU: the sparse GCN's ``wide_hidden`` option (``ggnn_gcn_config.wide_hidden``) through the host-only prepare calls at 132 SMs.

With it, hidden sizes up to 512 are accepted and every hidden size above 128 on bf16x3 / bf16 plans the streaming wgmma path: fixed
128-row tiles, two launches per layer (a weighted gather into the operand image, then the TMA-fed streaming GEMM).  At hidden <= 128 the
option changes nothing, byte for byte; fp32 keeps its CUDA-core kernel.  Dataset batches plan like the edge-list builder with it, the
plug-in option reaches the engine without changing params, and the GGNN plug-ins refuse it."""
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GgnnError, PreparedGraph
from tests import gcn_oracle as G
from tests.test_device_data_cpu import batch_ids, gcn_graph_set, packed_graph, plan_of, tile_starts
from tests.test_forward_plans_cpu import stream_ksteps

NUM_SMS = 132
L = 3
WIDE = [132, 160, 192, 256, 260, 288, 384, 512]
PLAN_RE = re.compile(r"^gcn-stream-(bf16x3|bf16) \(2 launches per layer: weighted gather, GEMM\) tiles=(\d+) DP=(\d+) N-blocks=(\d+)x128$")


def _graph(V=300, nnz=1500, seed=0):
    rng = np.random.default_rng(seed)
    lst, w = G.random_gcn_list(V, nnz, rng, isolated=(0, 5))
    return V, lst, w


def _prep(D, precision, wide, V, lst, w, **kw):
    return PreparedGraph.host_only_gcn(D, L, V, lst, w, use_bias=True, precision=precision, num_sms=NUM_SMS, wide_hidden=wide, **kw)


def stream_instance(plan):
    """The streaming kernel instance a gcn-stream plan launches: ``("stream", X3, KS)``, as forward_gcn_stream picks it."""
    m = PLAN_RE.match(plan)
    assert m, plan
    return ("stream", m.group(1) == "bf16x3", stream_ksteps(int(m.group(3)), {}))


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("D", WIDE)
def test_wide_hidden_plans_the_streaming_gcn(D, precision, monkeypatch):
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM", "GGNN_TS_KSTEPS"):
        monkeypatch.delenv(k, raising=False)
    V, lst, w = _graph(seed=D)
    g = _prep(D, precision, True, V, lst, w)
    info = g.info()
    m = PLAN_RE.match(info["plan"])
    assert m, info["plan"]
    DP = (D + 15) // 16 * 16
    ntiles = (V + 127) // 128
    assert (m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))) == (precision, ntiles, DP, (DP + 127) // 128)
    assert info["num_tiles"] == ntiles and not info["streaming"]   # no pair tables: the gather reads the target CSR
    np.testing.assert_array_equal(g.arrays(1)["tile_start"], list(range(0, V, 128)) + [V])
    with pytest.raises(GgnnError):
        g.stream_tables()


def test_the_widths_reach_every_stream_instance():
    from tests.test_forward_plans_cpu import inventory
    V, lst, w = _graph()
    seen = {stream_instance(_prep(D, p, True, V, lst, w).info()["plan"]) for D in WIDE for p in ("bf16x3", "bf16")}
    assert seen == {("stream", x3, ks) for x3, ks in inventory()["stream"]}, seen


def test_limits_with_the_option():
    V, lst, w = _graph()
    assert PLAN_RE.match(_prep(512, "bf16x3", True, V, lst, w).info()["plan"])
    assert _prep(512, "fp32", True, V, lst, w).info()["plan"].startswith("gcn-fp32-ffma GLOBAL(")
    assert _prep(260, "fp32", True, V, lst, w).info()["plan"].startswith("gcn-fp32-ffma GLOBAL(")
    for precision in ("bf16x3", "bf16", "fp32"):
        with pytest.raises(GgnnError, match="hidden_size > 512"):
            _prep(516, precision, True, V, lst, w)
    # without it, as before: 256 on the fp32 kernel, 260 refused
    assert _prep(256, "bf16x3", False, V, lst, w).info()["plan"].startswith("gcn-fp32-ffma")
    with pytest.raises(GgnnError, match="hidden_size > 256"):
        _prep(260, "bf16x3", False, V, lst, w)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "fp32"])
@pytest.mark.parametrize("D", [4, 16, 100, 128])
@pytest.mark.parametrize("save", [False, True])
def test_up_to_128_the_option_changes_nothing(D, precision, save):
    rng = np.random.default_rng(D)
    Vc, lc, wc = G.component_list(list(rng.integers(5, 30, 60)), rng)   # LOCAL tiles
    for V, lst, w in ((Vc, lc, wc), _graph(seed=D)):                   # one big component: GLOBAL
        a, b = _prep(D, precision, False, V, lst, w, save_for_backward=save), _prep(D, precision, True, V, lst, w, save_for_backward=save)
        assert a.info() == b.info()
        np.testing.assert_array_equal(a.image(), b.image())


@pytest.mark.parametrize("hidden,precision", [(256, "bf16x3"), (512, "bf16"), (384, "fp32"), (100, "bf16x3")])
@pytest.mark.parametrize("save", [False, True])
def test_dataset_batches_plan_like_the_edge_list_builder(hidden, precision, save):
    flat = packing.FlatGCNGraphs(gcn_graph_set())
    ds = DeviceDataset.host_only_gcn(hidden, L, flat, precision=precision, num_sms=NUM_SMS, for_training=save, wide_hidden=True)
    for ids in batch_ids(flat.num_graphs, seed=hidden):
        b = ds.prepare_batch(ids, save_for_backward=save)
        packed = packed_graph(flat, ids, hidden)
        ref = PreparedGraph.host_only_gcn(hidden, L, packed["initial_node_representation"].shape[0], packed["adjacency_list"],
                                          packed["adjacency_weights"], precision=precision, num_sms=NUM_SMS, save_for_backward=save,
                                          wide_hidden=True)
        got, want = b.info(), ref.info()
        assert plan_of(got) == plan_of(want), ids
        if hidden > 128 and precision != "fp32" and len(ids):
            assert want["plan"].startswith("gcn-stream-"), want["plan"]
        np.testing.assert_array_equal(got["tile_start"], tile_starts(ref, 1))


def test_dataset_without_the_option_refuses_wide_hidden_sizes():
    flat = packing.FlatGCNGraphs(gcn_graph_set(4))
    with pytest.raises(GgnnError, match="hidden_size > 256"):
        DeviceDataset.host_only_gcn(384, L, flat, precision="bf16x3")


# ---------------------------------------------------------------------------------------------------------------- plug-ins
def _plugin_args(tmp_path, **extra):
    mols = synthetic.make_molecules(30, seed=1)
    args = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:20], "--valid_data": mols[20:],
            "--config": {"hidden_size": 510, "batch_size": 200, "num_timesteps": 2, "num_epochs": 1}}
    args.update(extra)
    return args


def test_plugin_passes_the_option_to_the_engine(tmp_path, monkeypatch):
    from gated_graph_neural_network_samples_b200 import chem_gcn
    from tests.test_chem_gcn_cpu import StandInGCNEngine, StandInPropagation
    seen = []

    class Recording(StandInGCNEngine):
        def __init__(self, hidden_size, num_layers, use_bias=False, device=0, precision="fp32", **kw):
            seen.append((hidden_size, precision, kw))
            super().__init__(hidden_size, num_layers, use_bias, device, precision)

    monkeypatch.setattr(chem_gcn, "GCNEngine", Recording)
    monkeypatch.setattr(chem_gcn, "_propagation_function", lambda: StandInPropagation)
    a = chem_gcn.SparseGCNChemModel(_plugin_args(tmp_path, **{"--precision": "bf16x3", "--gcn-wide-hidden": True}))
    b = chem_gcn.SparseGCNChemModel(_plugin_args(tmp_path, **{"--precision": "bf16x3"}))
    # 510 is not a multiple of 4: the engine runs zero-padded at 512
    assert seen == [(512, "bf16x3", {"wide_hidden": True}), (512, "bf16x3", {})]
    assert a.params == b.params   # a command-line option, not a params key: checkpoints move between the two
    assert a.weights["edge_weights"][0].shape == (510, 510)


def test_ggnn_plugins_refuse_the_option(tmp_path):
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    args = _plugin_args(tmp_path, **{"--gcn-wide-hidden": True})
    args["--config"] = {"hidden_size": 16, "batch_size": 8}
    for cls in (SparseGGNNChemModel, DenseGGNNChemModel):
        with pytest.raises(Exception, match="--gcn-wide-hidden applies to the sparse GCN model"):
            cls(args)


# ---------------------------------------------------------------------------------------------------------------- the oracle
def test_oracle_statements_agree_at_512():
    import torch
    rng = np.random.default_rng(5)
    D, Lo, V = 512, 3, 40
    lst, w = G.random_gcn_list(V, 200, rng, isolated=(3,))
    ks = [G.glorot((D, D), rng) for _ in range(Lo)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(Lo)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    masks = [(rng.random((V, D)) < 0.8).astype(np.float32) for _ in range(Lo - 1)]
    a = G.gcn_propagation_loops(h0, lst, w, ks, bs, masks, 0.8)
    b = G.gcn_propagation_torch(torch.from_numpy(h0).double(), lst, torch.from_numpy(w).double(), [torch.from_numpy(k).double() for k in ks],
                                [torch.from_numpy(x).double() for x in bs], masks, 0.8).numpy()
    np.testing.assert_allclose(a, b, rtol=1e-10, atol=1e-10 * np.abs(a).max())
