"""CPU: the dense model's adjacency as a device tensor (ggnn_prepare_graph_dense_device, DESIGN §2.14) without a GPU -- the ABI, the
host-only prepare (plan texts at every precision and the hidden sizes that pick different plans, the value-independent streaming tables,
the same image bytes at every host-thread count, refusals, an empty batch), the float64 statement of dA against float64 autograd, and the
dense plug-in's choice of route (a torch tensor feed: the device batch and the adjacency's gradient; a NumPy feed: today's host path)."""
import os
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import _lib, chem_dense, synthetic
from oracle import ggnn_oracle as O
from tests import dense_adjacency_oracle as DA
from tests.test_chem_model_cpu import StandInEngine
from tests.test_deterministic_cpu import RecordingEngine

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ggnn_b200.h")
TAG = " [dense adjacency on the device]"


def _lib_or_skip():
    try:
        return _lib.load()
    except Exception as ex:   # the library is built by build(); without nvcc and without a built library there is nothing to call
        pytest.skip("libggnn_b200.so unavailable: %s" % ex)


def _params(D, **kw):
    p = {"hidden_size": D, "layer_timesteps": [2], "residual_connections": {}, "use_edge_bias": True,
         "use_edge_msg_avg_aggregation": False, "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}
    p.update(kw)
    return p


def _host(D, precision, b=3, v=29, T=4, save=True, **kw):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    _lib_or_skip()
    return PreparedGraph.host_only_dense_device(_params(D, **kw), T, b, v, precision=precision, save_for_backward=save)


def test_header_declares_and_lib_binds_the_new_calls():
    import ctypes as C
    text = open(HEADER).read()
    assert re.search(r"int ggnn_prepare_graph_dense_device\(const ggnn_engine\* e, int32_t save_for_backward, int32_t num_graphs, "
                     r"int32_t num_vertices,\s+ggnn_prepared_graph\*\* inout\);", text)
    assert re.search(r"int ggnn_host_prepare_graph_dense_device\(const ggnn_config\* cfg, int32_t num_sms, int32_t save_for_backward, "
                     r"int32_t num_graphs,\s+int32_t num_vertices, ggnn_prepared_graph\*\* inout\);", text)
    assert _lib.SYMBOLS["ggnn_prepare_graph_dense_device"] == (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)])
    assert _lib.SYMBOLS["ggnn_host_prepare_graph_dense_device"][1][0] == C.POINTER(_lib.GgnnConfig)
    lib = _lib_or_skip()
    for name in ("ggnn_prepare_graph_dense_device", "ggnn_host_prepare_graph_dense_device"):
        getattr(lib, name)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "fp32"])
@pytest.mark.parametrize("D", [4, 100, 128, 132, 256, 512])
def test_plan_text_and_value_independent_tables(precision, D):
    b, v, T = 3, 29, 4
    g = _host(D, precision, b, v, T)
    info = g.info()
    V = b * v
    assert info["num_nodes"] == V and info["num_messages"] == b * T * v * v
    assert info["plan"].endswith(TAG), info["plan"]
    a = g.arrays(T)
    np.testing.assert_array_equal(a["row_ptr"], 0)                              # the image lists no messages
    np.testing.assert_array_equal(a["tile_start"], np.minimum(np.arange(info["num_tiles"] + 1) * 128, V))
    if precision == "fp32":
        assert info["plan"].startswith("fp32-stepwise ") and not info["streaming"], info["plan"]
        return
    assert info["plan"].startswith("wgmma-%s STREAM(4 launches per step: dense aggregation" % precision), info["plan"]
    assert info["streaming"]
    pair = a["pair_src"]
    want = np.full(info["num_tiles"] * 128 * T, -1, np.int64)
    want[:V * T] = -(2 + np.arange(V * T))                                        # every (row, type) pair is virtual row row*T + type
    np.testing.assert_array_equal(pair, want)
    st = g.stream_tables()
    np.testing.assert_array_equal(st["tile_vptr"], 0)                             # an empty range for every tile: the prologue sums nothing
    assert st["vrow_ptr"].shape[0] == V * T + 1 and st["vsrc"].shape[0] == 0 and st["vslot"] is None
    np.testing.assert_array_equal(st["vrow_ptr"], 0)


def test_tile_masks_have_every_type():
    """The streaming plan's per-tile edge-type masks (the image section after the tile starts) have all T bits set."""
    for T in (1, 4, 32):
        g = _host(256, "bf16x3", b=10, v=29, T=T)
        img = g.image().view(np.uint8)
        nt = g.info()["num_tiles"]
        ts = np.frombuffer(img.tobytes(), np.int32)
        # tile_start is the only run of nt + 1 int32 0, 128, ..., V in the image; the masks follow at the next 16-byte boundary
        starts = np.minimum(np.arange(nt + 1) * 128, 290).astype(np.int32)
        pos = next(i for i in range(ts.shape[0] - nt) if np.array_equal(ts[i:i + nt + 1], starts))
        off = (pos * 4 + (nt + 1) * 4 + 15) // 16 * 16
        masks = np.frombuffer(img.tobytes()[off:off + 4 * nt], np.uint32)
        np.testing.assert_array_equal(masks, np.uint32((1 << T) - 1 if T < 32 else 0xFFFFFFFF))


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_image_bytes_at_every_host_thread_count(precision, monkeypatch):
    ref = None
    for n in range(1, 9):
        monkeypatch.setenv("GGNN_HOST_THREADS", str(n))
        img = _host(260 if precision == "fp32" else 256, precision, b=64, v=29).image()
        if ref is None:
            ref = img
        np.testing.assert_array_equal(img, ref)


def test_refusals_and_the_empty_batch():
    from gated_graph_neural_network_samples_b200.engine import GgnnError, PreparedGraph
    _lib_or_skip()
    with pytest.raises(GgnnError, match="attention"):
        PreparedGraph.host_only_dense_device(_params(100, use_propagation_attention=True), 4, 2, 29, precision="fp32")
    with pytest.raises(GgnnError, match="use_edge_msg_avg_aggregation"):
        PreparedGraph.host_only_dense_device(_params(100, use_edge_msg_avg_aggregation=True), 4, 2, 29, precision="bf16x3")
    with pytest.raises(GgnnError, match="CudnnCompatibleGRUCell"):
        PreparedGraph.host_only_dense_device(_params(100, graph_rnn_cell="CudnnCompatibleGRUCell"), 4, 2, 29, precision="bf16x3",
                                             cudnn_gru_tensor_cores=True)
    with pytest.raises(GgnnError):
        PreparedGraph.host_only_dense_device(_params(100), 4, 2, 0, precision="fp32")
    for precision in ("bf16x3", "fp32"):
        g = _host(100, precision, b=0, v=29)
        info = g.info()
        assert info["num_nodes"] == 0 and info["num_messages"] == 0 and info["num_tiles"] == 0 and info["plan"].endswith(TAG)


# ---------------------------------------------------------------------------------------------------------------- the gradient statement
def _soft(b, T, v, rng):
    s = rng.normal(0, 1, (b, T, v, v))
    e = np.exp(s - s.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def test_adjacency_grad_statement_equals_float64_autograd_of_the_dense_oracle():
    import torch
    rng = np.random.default_rng(4)
    b, T, v, D = 3, 4, 7, 12
    dp = {"hidden_size": D, "num_timesteps": 3, "use_edge_bias": True}
    w = O.init_dense_weights(dp, T, rng)
    h0 = rng.normal(0, 0.5, (b, v, D))
    A = torch.tensor(_soft(b, T, v, rng) - 0.1, dtype=torch.float64, requires_grad=True)   # negative entries too
    g = torch.tensor(rng.normal(0, 1, (b, v, D)))
    out = O.dense_propagation_torch(h0, A, w, dp, dtype=torch.float64)
    (out * g).sum().backward()
    record = []
    A2 = A.detach().clone().requires_grad_(True)
    ew = dict(w, edge_biases=w["edge_biases"].reshape(T, D))
    mine = DA.propagation_torch(h0.reshape(b * v, D), A2, [ew], _params(D, layer_timesteps=[3]), record=record)
    np.testing.assert_allclose(mine.detach().numpy().reshape(b, v, D), out.detach().numpy(), rtol=1e-12, atol=1e-12)
    (mine.reshape(b, v, D) * g).sum().backward()
    stmt = DA.adjacency_grad_statement(record, b, v)
    np.testing.assert_allclose(stmt.numpy(), A.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(A2.grad.numpy(), A.grad.numpy(), rtol=1e-10, atol=1e-12)


def test_adjacency_grad_statement_multi_layer_rnn_with_residual():
    import torch
    rng = np.random.default_rng(5)
    b, T, v, D = 2, 3, 5, 8
    p = _params(D, layer_timesteps=[2, 1], residual_connections={"1": [0]}, graph_rnn_cell="RNN", graph_rnn_activation="relu")
    w = O.init_sparse_weights(p, T, rng, edge_bias_scale=0.3)
    A = torch.tensor(rng.normal(0, 1, (b, T, v, v)), requires_grad=True)
    record = []
    out = DA.propagation_torch(rng.normal(0, 0.5, (b * v, D)), A, w, p, record=record)
    (out * torch.tensor(rng.normal(0, 1, out.shape))).sum().backward()
    np.testing.assert_allclose(DA.adjacency_grad_statement(record, b, v).numpy(), A.grad.numpy(), rtol=1e-10, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------------- the plug-in's route
class DeviceRecordingEngine(RecordingEngine):
    """The recording stand-in engine with the calls of a dense-device batch: the identity propagation of RecordingEngine, dA = 1."""

    def prepare_graph_dense_device(self, num_graphs, num_vertices, save_for_backward=None, reuse=None):
        self.calls.append(("prepare_graph_dense_device", num_graphs, num_vertices))
        return ("prepared", num_graphs, num_vertices)

    def set_graph_prepared(self, g):
        self.calls.append(("set_graph_prepared", g))

    def set_message_weights(self, w):
        self.calls.append(("set_message_weights", tuple(w.shape)))

    def set_graph_dense(self, adjacency_matrix):
        self.calls.append(("set_graph_dense",))
        StandInEngine.set_graph_dense(self, adjacency_matrix)

    def backward(self, d_out, grads, d_h0, d_message_weights=None):
        self.calls.append(("backward", d_message_weights is not None))
        if d_h0 is not None:
            d_h0.copy_(d_out)
        if d_message_weights is not None:
            d_message_weights.fill_(1.0)


def _dense_model(tmp_path, monkeypatch):
    monkeypatch.setattr(chem_dense, "PropagationEngine", DeviceRecordingEngine)
    mols = synthetic.make_molecules(16, seed=1)
    m = chem_dense.DenseGGNNChemModel({"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:12], "--valid_data": mols[12:],
                                       "--config": {"hidden_size": 16, "batch_size": 4, "num_timesteps": 2}})
    feed = next(iter(m.make_minibatch_iterator(m.train_data, True)))
    feed.pop("_prepared_graph", None)
    return m, feed


def test_plugin_takes_the_device_route_for_a_tensor_feed(tmp_path, monkeypatch):
    import torch
    m, feed = _dense_model(tmp_path, monkeypatch)
    adj = np.asarray(feed["adjacency_matrix"], np.float32)
    scale = torch.tensor(0.5, requires_grad=True)
    feed["adjacency_matrix"] = torch.from_numpy(adj) * scale                  # a computed adjacency: its producer gets the gradient
    m.feed = feed
    m.compute_final_node_representations().sum().backward()
    names = [c[0] for c in m.engine.calls]
    b, _, v, _ = adj.shape
    assert ("prepare_graph_dense_device", b, v) in m.engine.calls and "set_graph_prepared" in names and "set_graph_dense" not in names
    assert ("set_message_weights", adj.shape) in m.engine.calls and ("backward", True) in m.engine.calls
    assert float(scale.grad) == pytest.approx(float(adj.sum()))                # dA = 1 from the stand-in: d scale = sum(adj)


def test_plugin_keeps_the_host_route_for_a_numpy_feed(tmp_path, monkeypatch):
    m, feed = _dense_model(tmp_path, monkeypatch)
    m.feed = feed
    m.compute_final_node_representations().sum().backward()
    names = [c[0] for c in m.engine.calls]
    assert "set_graph_dense" in names and "prepare_graph_dense_device" not in names and "set_message_weights" not in names
    assert ("backward", False) in m.engine.calls


# ---------------------------------------------------------------------------------------------------------------- the kernels
def test_new_kernels_use_no_stack_and_do_not_spill():
    """The five kernels of ggnn_dense_adj.cuh (three dense_apply_kernel instances, dense_adj_grad_kernel, dense_row_sums_kernel):
    no stack frame, no local memory."""
    import shutil
    import subprocess
    exe = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(exe):
        pytest.skip("cuobjdump is not available")
    from gated_graph_neural_network_samples_b200 import _build
    _lib_or_skip()
    out = subprocess.run([exe, "-res-usage", _build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1) if "4dadj" in m.group(1) else None
            continue
        if name is not None and "REG:" in line:
            found[name] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            name = None
    assert len(found) == 5, sorted(found)
    for k, r in found.items():
        assert r["STACK"] == 0 and r.get("LOCAL", 0) == 0, (k, r)
