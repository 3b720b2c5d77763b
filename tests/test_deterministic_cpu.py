"""CPU: deterministic mode without a GPU -- ``ggnn_set_deterministic`` is declared and bound, refuses NULL, and the autograd nodes of the
sparse, dense and GCN plug-ins pass ``torch.are_deterministic_algorithms_enabled()`` to the engine before every engine call, on and off.
The plug-ins are driven with the stand-in engines of tests/test_chem_model_cpu.py and tests/test_chem_gcn_cpu.py, extended with the engine
calls the real autograd nodes make."""
import os
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import _lib, chem_dense, chem_gcn, chem_sparse, synthetic
from gated_graph_neural_network_samples_b200.readout import gated_readout_function
from tests.test_chem_gcn_cpu import StandInGCNEngine, StandInPropagation as GCNStandInPropagation
from tests.test_chem_model_cpu import StandInEngine, StandInPropagation

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ggnn_b200.h")


def test_header_declares_and_lib_binds_set_deterministic():
    text = open(HEADER).read()
    assert re.search(r"int ggnn_set_deterministic\(ggnn_engine\* e, int32_t enable\);", text)
    import ctypes as C
    assert _lib.SYMBOLS["ggnn_set_deterministic"] == (C.c_int, [C.c_void_p, C.c_int32])


def test_set_deterministic_refuses_null():
    try:
        lib = _lib.load()
    except Exception as ex:   # the library is built by build(); without nvcc and without a built library there is nothing to call
        pytest.skip("libggnn_b200.so unavailable: %s" % ex)
    assert lib.ggnn_set_deterministic(None, 1) == -1   # GGNN_EINVAL
    assert lib.ggnn_set_deterministic(None, 0) == -1


class _Recorder:
    """The engine calls of the real autograd nodes, recorded: set_deterministic's flag in order, around forward / backward."""

    def _init_recorder(self):
        self.calls, self.serial = [], 0

    def set_deterministic(self, enable):
        self.calls.append(("det", bool(enable)))

    def set_weights(self, *a, **k):
        self.serial += 1

    def require_serial(self, serial, what=""):
        assert serial == self.serial


class RecordingEngine(StandInEngine, _Recorder):
    """The GGNN stand-in engine with the forward / backward the real autograd node calls (identity propagation: only the calls matter)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self._init_recorder()

    def forward(self, h0):
        self.calls.append(("forward",))
        self._h0 = h0
        return h0.clone()

    def backward(self, d_out, grads, d_h0):
        self.calls.append(("backward",))
        if d_h0 is not None:
            d_h0.copy_(d_out)


class RecordingGCNEngine(StandInGCNEngine, _Recorder):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self._init_recorder()

    def forward(self, h0):
        self.calls.append(("forward",))
        return h0.clone()

    def backward(self, d_out, grads, d_h0):
        self.calls.append(("backward",))
        if d_h0 is not None:
            d_h0.copy_(d_out)


def _flags_before(calls, what):
    """The flag set by the last set_deterministic before every ``what`` call."""
    out, flag = [], None
    for c in calls:
        if c[0] == "det":
            flag = c[1]
        elif c[0] == what:
            out.append(flag)
    return out


@pytest.fixture(params=[False, True], ids=["flag-off", "flag-on"])
def det_flag(request):
    import torch
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev)


def _one_training_batch(m):
    m.feed = next(iter(m.make_minibatch_iterator(m.train_data, True)))
    m.compute_final_node_representations().sum().backward()


@pytest.mark.parametrize("plugin", ["sparse", "dense"])
def test_ggnn_plugins_pass_the_torch_flag_to_the_engine(tmp_path, monkeypatch, det_flag, plugin):
    monkeypatch.setattr(chem_sparse, "PropagationEngine", RecordingEngine)
    monkeypatch.setattr(chem_dense, "PropagationEngine", RecordingEngine)
    mols = synthetic.make_molecules(16, seed=1)
    if plugin == "sparse":
        cfg = {"hidden_size": 16, "batch_size": 300, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}}
        m = chem_sparse.SparseGGNNChemModel({"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:12],
                                             "--valid_data": mols[12:], "--config": cfg})
    else:
        cfg = {"hidden_size": 16, "batch_size": 4, "num_timesteps": 2}
        m = chem_dense.DenseGGNNChemModel({"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:12],
                                           "--valid_data": mols[12:], "--config": cfg})
    assert m._propagation is not StandInPropagation
    _one_training_batch(m)
    calls = m.engine.calls
    assert _flags_before(calls, "forward") == [det_flag] and _flags_before(calls, "backward") == [det_flag], calls


def test_gcn_plugin_passes_the_torch_flag_to_the_engine(tmp_path, monkeypatch, det_flag):
    monkeypatch.setattr(chem_gcn, "GCNEngine", RecordingGCNEngine)
    mols = synthetic.make_molecules(16, seed=1)
    m = chem_gcn.SparseGCNChemModel({"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:12], "--valid_data": mols[12:],
                                     "--config": {"hidden_size": 16, "batch_size": 300, "num_timesteps": 2, "gcn_use_bias": True}})
    assert m._propagation is not GCNStandInPropagation
    _one_training_batch(m)
    calls = m.engine.calls
    assert _flags_before(calls, "forward") == [det_flag] and _flags_before(calls, "backward") == [det_flag], calls


def test_readout_node_passes_the_torch_flag_to_the_engine(det_flag):
    import torch

    class ReadoutEngine(_Recorder):
        def readout_forward(self, h_last, h0, w_gate, b_gate, w_trans, b_trans):
            self.calls.append(("forward",))
            return h_last.sum(1)

        def readout_backward(self, h_last, h0, w_gate, b_gate, w_trans, b_trans, d_out):
            self.calls.append(("backward",))
            D = h_last.shape[1]
            return (d_out[:, None].expand_as(h_last).clone(), torch.zeros(2 * D), torch.zeros(1), torch.zeros(D), torch.zeros(1))

    eng = ReadoutEngine()
    eng._init_recorder()
    D = 8
    h = torch.randn(5, D, requires_grad=True)
    w = [torch.randn(2 * D, 1, requires_grad=True), torch.zeros(1, requires_grad=True), torch.randn(D, 1, requires_grad=True),
         torch.zeros(1, requires_grad=True)]
    gated_readout_function().apply(eng, h, torch.randn(5, D), *w).sum().backward()
    assert _flags_before(eng.calls, "forward") == [det_flag] and _flags_before(eng.calls, "backward") == [det_flag], eng.calls
    np.testing.assert_array_equal(h.grad.numpy(), np.ones((5, D), np.float32))
