"""CPU: the bf16x3 tensor-core backward's surface without a GPU -- the C ABI declaration and binding of
``ggnn_set_backward_precision``, the ``--backward-precision`` argument of the three plug-ins (against recording stand-in engines), and
what ptxas made of the new kernels (``cuobjdump -res-usage`` of the built library: registers pinned, no local-memory spills)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import chem_dense, chem_gcn, chem_sparse, synthetic
from tests.test_chem_gcn_cpu import StandInGCNEngine, StandInPropagation as GCNPropagation
from tests.test_chem_model_cpu import StandInEngine, StandInPropagation

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ggnn_b200.h")


def test_header_declares_and_lib_binds_the_setting():
    import ctypes as C
    from gated_graph_neural_network_samples_b200 import _lib
    with open(HEADER) as f:
        text = f.read()
    assert re.search(r"int ggnn_set_backward_precision\(ggnn_engine\* e, int32_t precision\);", text)
    assert _lib.SYMBOLS["ggnn_set_backward_precision"] == (C.c_int, [C.c_void_p, C.c_int32])
    lib = _lib.load()
    assert lib.ggnn_set_backward_precision(None, 0) == -1      # GGNN_EINVAL: no engine
    assert lib.ggnn_set_backward_precision(None, 1) == -1


def test_python_engine_refuses_unknown_names_before_the_abi():
    from gated_graph_neural_network_samples_b200.engine import BACKWARD_PRECISIONS, PRECISIONS, PropagationEngine
    assert BACKWARD_PRECISIONS == ("fp32", "bf16x3") and [PRECISIONS[p] for p in BACKWARD_PRECISIONS] == [0, 1]
    stub = PropagationEngine.__new__(PropagationEngine)        # no device: the name check comes first
    for bad in ("bf16", "fp16", ""):
        with pytest.raises(ValueError):
            stub.set_backward_precision(bad)


# ---------------------------------------------------------------------------------------------------------------- the plug-ins
class RecordingEngine(StandInEngine):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.bwd = []

    def set_backward_precision(self, precision):
        self.bwd.append(precision)


class RecordingGCNEngine(StandInGCNEngine):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.bwd = []

    def set_backward_precision(self, precision):
        self.bwd.append(precision)


@pytest.fixture
def recording(monkeypatch):
    monkeypatch.setattr(chem_sparse, "PropagationEngine", RecordingEngine)
    monkeypatch.setattr(chem_sparse, "_propagation_function", lambda: StandInPropagation)
    monkeypatch.setattr(chem_dense, "PropagationEngine", RecordingEngine)
    monkeypatch.setattr(chem_dense, "_propagation_function", lambda: StandInPropagation)
    monkeypatch.setattr(chem_gcn, "GCNEngine", RecordingGCNEngine)
    monkeypatch.setattr(chem_gcn, "_propagation_function", lambda: GCNPropagation)


PLUGINS = {
    "sparse": (lambda a: chem_sparse.SparseGGNNChemModel(a), {"hidden_size": 16, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}}),
    "dense": (lambda a: chem_dense.DenseGGNNChemModel(a), {"hidden_size": 16, "num_timesteps": 2, "batch_size": 8}),
    "gcn": (lambda a: chem_gcn.SparseGCNChemModel(a), {"hidden_size": 16, "num_timesteps": 2}),
}


def _args(tmp_path, cfg, **extra):
    mols = synthetic.make_molecules(24, seed=1)
    return dict({"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:16], "--valid_data": mols[16:],
                 "--config": dict({"batch_size": 300, "num_epochs": 1}, **cfg)}, **extra)


@pytest.mark.parametrize("kind", sorted(PLUGINS))
def test_plugins_pass_the_argument_to_their_engine(kind, tmp_path, recording):
    make, cfg = PLUGINS[kind]
    for given in ("bf16x3", "fp32"):
        m = make(_args(tmp_path, cfg, **{"--backward-precision": given}))
        assert m.backward_precision == given and m.engine.bwd == [given]
        assert np.isfinite(m.run_epoch("train", m.train_data, True)[0])


@pytest.mark.parametrize("kind", sorted(PLUGINS))
def test_plugins_make_no_call_without_the_argument(kind, tmp_path, recording):
    make, cfg = PLUGINS[kind]
    m = make(_args(tmp_path, cfg))
    assert m.backward_precision is None and m.engine.bwd == []


@pytest.mark.parametrize("bad", ["bf16", "BF16X3", "fp64"])
@pytest.mark.parametrize("kind", sorted(PLUGINS))
def test_plugins_refuse_unknown_names_before_any_engine(kind, bad, tmp_path, monkeypatch):
    made = []
    for mod, name in ((chem_sparse, "PropagationEngine"), (chem_dense, "PropagationEngine"), (chem_gcn, "GCNEngine")):
        monkeypatch.setattr(mod, name, lambda *a, **k: made.append(a))
    make, cfg = PLUGINS[kind]
    with pytest.raises(Exception, match="Unknown backward precision"):
        make(_args(tmp_path, cfg, **{"--backward-precision": bad}))
    assert made == []


# ---------------------------------------------------------------------------------------------------------------- the binary
# ptxas's registers per thread of every new kernel instance, measured on the sm_90a build (CUDA 12.9).  The data-gradient kernel runs two
# 256-thread CTAs per SM (<= 128 registers), the weight-gradient kernels' 128-thread CTAs are limited by shared memory (32 KB each).
EXPECTED_REGS = {"gemm_nt_tc_kernelILb0E": 113, "gemm_nt_tc_kernelILb1E": 113, "gemm_tn_tc_atomic_kernel": 94, "gemm_tn_tc_split_kernel": 94}


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def test_kernel_registers_and_no_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump is not available")
    from gated_graph_neural_network_samples_b200 import _build, _lib
    _lib.load()
    out = subprocess.run([exe, "-res-usage", _build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found, key = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            key = next((k for k in EXPECTED_REGS if k in m.group(1) and "bwd_tc" in m.group(1)), None)
            continue
        if key is not None and "REG:" in line:
            found[key] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            key = None
    assert sorted(found) == sorted(EXPECTED_REGS), sorted(found)
    for k, regs in EXPECTED_REGS.items():
        assert found[k]["REG"] == regs, (k, found[k])
        assert found[k]["STACK"] == 0 and found[k].get("LOCAL", 0) == 0, (k, found[k])
