"""CPU-only: the readout map built from device arrays (``ggnn_readout_set_graphs_device``, DESIGN 2.17) -- the header declarations and
their documented promises, the exported symbols and their ctypes signatures, the NULL engine, the Python checks that refuse a bad feed
before any call (with a stand-in for CUDA tensors), the plug-ins' routes for host feeds, and the resources of the new kernels (no stack
frame, no spills).  Sections, bits and refusals against the host builder are in tests/test_gpu_readout_map_device.py."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    """The header with comment continuation marks (a line's leading ` * `) removed and whitespace collapsed."""
    with open(os.path.join(ROOT, "include", "ggnn_b200.h")) as f:
        return re.sub(r"\s+", " ", re.sub(r"\n\s*\*(?!/)", " ", f.read()))


def _block(h, name):
    """The header's comment block over the entry ``name``."""
    end = h.index("int %s(" % name)
    return h[h.rindex("/*", 0, end):end]


def _codes():
    return {k: int(v) for k, v in re.findall(r"(GGNN_E[A-Z]+) = (-?\d+)", _header())}


def test_header_declares_the_entries_and_documents_their_promises():
    h = _header()
    assert ("int ggnn_readout_set_graphs_device(ggnn_engine* e, int32_t num_nodes, const int32_t* graph_nodes_list, int32_t num_graphs, "
            "int32_t nodes_per_graph, const float* node_mask, ggnn_stream_t stream);") in h
    assert ("int ggnn_readout_map(ggnn_engine* e, int32_t* num_nodes, int32_t* num_graphs, int32_t* flags, int32_t* graph_of, int32_t* start, "
            "int32_t* perm, float* node_mask, ggnn_stream_t stream);") in h
    b = _block(h, "ggnn_readout_set_graphs_device")
    assert "ggnn_readout_set_graphs with graph_nodes_list [V] int32 and node_mask [V] fp32 in the engine's device memory" in b
    assert "synchronises `stream` once" in b
    assert "does not depend on the order of any atomic" in b
    assert "no node is copied to the host" in b
    assert "lowest out-of-range node" in b
    for code in ("GGNN_ERANGE", "GGNN_EINVAL", "GGNN_ESTATE"):
        assert code in b, code
    # the entry sits next to the host call it mirrors
    assert h.index("int ggnn_readout_set_graphs(") < h.index("int ggnn_readout_set_graphs_device(") < h.index("int ggnn_readout_forward(")


def test_symbols_are_exported_with_their_signatures():
    from gated_graph_neural_network_samples_b200 import _lib
    lib = _lib.load()
    fn = lib.ggnn_readout_set_graphs_device
    assert fn.restype is C.c_int
    assert fn.argtypes == [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    assert fn.argtypes == lib.ggnn_readout_set_graphs.argtypes
    m = lib.ggnn_readout_map
    assert m.restype is C.c_int
    assert m.argtypes == [C.c_void_p] + [C.POINTER(C.c_int32)] * 3 + [C.c_void_p] * 5


def test_null_engine_is_refused_without_a_device():
    from gated_graph_neural_network_samples_b200 import _lib
    lib = _lib.load()
    codes = _codes()
    assert lib.ggnn_readout_set_graphs_device(None, 0, None, 0, 1, None, None) == codes["GGNN_EINVAL"]
    assert lib.ggnn_readout_set_graphs_device(None, 4, C.c_void_p(16), 2, 0, None, None) == codes["GGNN_EINVAL"]
    assert lib.ggnn_readout_map(None, None, None, None, None, None, None, None, None) == codes["GGNN_EINVAL"]


# ---------------------------------------------------------------------------------------------------------------- Python checks
class _NoLibrary:
    """Stands in for the library: any call into it fails the test (the feed checks run before the call)."""

    def __getattr__(self, name):
        raise AssertionError("%s was called" % name)


def _bare_engine():
    """A PropagationEngine's Python half without a library handle: enough for the feed checks, which run before any call."""
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine.__new__(PropagationEngine)
    eng._h = C.c_void_p()
    eng.lib = _NoLibrary()
    eng.D, eng.T, eng.L, eng.device, eng.serial = 32, 2, 1, 0, 0
    return eng


def _fake_cuda(t, index=0):
    """A CPU tensor that says it is on cuda:``index`` -- a stand-in for a CUDA tensor on a machine without one."""
    import torch

    class FakeCuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True

        @property
        def device(self):
            return torch.device("cuda", index)

    return torch.Tensor._make_subclass(FakeCuda, t)


def test_feed_checks_refuse_before_the_call():
    """dtype, shape, contiguity, device, then the mask's length: every bad CUDA feed raises GgnnError before the library is touched."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    eng = _bare_engine()
    gnl = torch.zeros(6, dtype=torch.int32)
    cases = [
        (dict(graph_nodes_list=_fake_cuda(gnl.long())), "graph_nodes_list must be int32"),       # int64 is out (no narrowing)
        (dict(graph_nodes_list=_fake_cuda(gnl.float())), "graph_nodes_list must be int32"),
        (dict(graph_nodes_list=_fake_cuda(gnl.reshape(2, 3))), "graph_nodes_list must be [V]"),
        (dict(graph_nodes_list=_fake_cuda(torch.zeros(12, dtype=torch.int32)[::2])), "graph_nodes_list must be contiguous"),
        (dict(graph_nodes_list=_fake_cuda(gnl, 1)), "graph_nodes_list must be on cuda:0"),       # another device
        (dict(graph_nodes_list=_fake_cuda(gnl), node_mask=_fake_cuda(torch.ones(6, dtype=torch.float64))), "node_mask must be float32"),
        (dict(graph_nodes_list=_fake_cuda(gnl), node_mask=_fake_cuda(torch.ones(12)[::2])), "node_mask must be contiguous"),
        (dict(graph_nodes_list=_fake_cuda(gnl), node_mask=_fake_cuda(torch.ones(5))), "node_mask has 5 entries for 6 nodes"),
        (dict(nodes_per_graph=4, node_mask=_fake_cuda(torch.ones(3, 4))), "node_mask has 12 entries for 8 nodes"),    # 2 graphs of 4
        (dict(nodes_per_graph=2, node_mask=_fake_cuda(torch.ones(2, 2), 1)), "node_mask must be on cuda:0"),
        (dict(nodes_per_graph=2, node_mask=_fake_cuda(torch.ones(4, dtype=torch.bool))), "node_mask must be float32"),
        # host and CUDA arguments do not mix, in either order
        (dict(graph_nodes_list=_fake_cuda(gnl), node_mask=np.ones(6, np.float32)), "must both be CUDA tensors or both host arrays"),
        (dict(graph_nodes_list=np.zeros(6, np.int32), node_mask=_fake_cuda(torch.ones(6))), "must both be CUDA tensors or both host arrays"),
        (dict(graph_nodes_list=gnl, node_mask=_fake_cuda(torch.ones(6))), "must both be CUDA tensors or both host arrays"),
    ]
    for kw, text in cases:
        with pytest.raises(GgnnError, match=re.escape(text)):
            eng.readout_set_graphs(2, **kw)
    assert not hasattr(eng, "_readout_shape")   # no refused call set a map


class _Recorder:
    """Stands in for the library and records the readout calls with their arguments."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            return 0
        return call


def test_host_values_take_the_host_entry_unchanged():
    """NumPy arrays, lists and CPU tensors go to ggnn_readout_set_graphs as contiguous int32 / fp32 host arrays, as before."""
    import torch
    eng = _bare_engine()
    eng.lib = _Recorder()
    eng._stream = lambda: 0
    gnl = np.array([0, 0, 1, 2, 2], np.int64)
    for feed in (gnl, list(gnl), torch.from_numpy(gnl.astype(np.int32))):
        eng.lib.calls.clear()
        eng.readout_set_graphs(3, graph_nodes_list=feed)
        [(name, args)] = eng.lib.calls
        assert name == "ggnn_readout_set_graphs" and args[1] == 5 and args[3] == 3 and args[5] is None
        kept = eng._readout_keepalive[0]
        assert kept.dtype == np.int32 and kept.ctypes.data == args[2]
        np.testing.assert_array_equal(kept, gnl)
    mask = np.ones((2, 3), np.float64)
    eng.lib.calls.clear()
    eng.readout_set_graphs(2, nodes_per_graph=3, node_mask=mask)
    [(name, args)] = eng.lib.calls
    assert name == "ggnn_readout_set_graphs" and args[1] == 6 and args[2] is None and args[4] == 3
    assert eng._readout_keepalive[1].dtype == np.float32 and eng._readout_shape == (6, 2)


def _plugin_shell(cls, feed, placeholders):
    """A plug-in's Python half around a recording engine: enough for _set_readout_map."""
    m = cls.__new__(cls)
    m.feed, m.placeholders = feed, placeholders
    m.engine = _bare_engine()
    m.engine.lib = _Recorder()
    m.engine._stream = lambda: 0
    return m


def test_plugins_route_host_values_to_the_host_entry():
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    gnl = np.array([0, 1, 1, 3], np.int32)
    for cls in (SparseGGNNChemModel, SparseGCNChemModel):
        m = _plugin_shell(cls, {"num_graphs": 4, "graph_nodes_list": gnl}, {"num_graphs": "num_graphs", "graph_nodes_list": "graph_nodes_list"})
        m._set_readout_map()
        [(name, args)] = m.engine.lib.calls
        assert name == "ggnn_readout_set_graphs" and args[1:2] == (4,) and args[3] == 4, cls
        np.testing.assert_array_equal(m.engine._readout_keepalive[0], gnl)
    mask = np.array([[1, 1, 0], [1, 0, 0]], np.float32)
    m = _plugin_shell(DenseGGNNChemModel, {"node_mask": mask}, {"node_mask": "node_mask"})
    m._set_readout_map()
    [(name, args)] = m.engine.lib.calls
    assert name == "ggnn_readout_set_graphs" and args[1] == 6 and args[2] is None and args[3] == 2 and args[4] == 3
    np.testing.assert_array_equal(m.engine._readout_keepalive[1], mask.reshape(-1))


def test_plugins_pass_cuda_values_through():
    """A CUDA list or mask reaches the device entry's checks as it is (here a stand-in on another device, refused by them)."""
    import torch
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    m = _plugin_shell(SparseGGNNChemModel, {"num_graphs": 2, "graph_nodes_list": _fake_cuda(torch.zeros(3, dtype=torch.int32), 1)},
                      {"num_graphs": "num_graphs", "graph_nodes_list": "graph_nodes_list"})
    with pytest.raises(GgnnError, match="graph_nodes_list must be on cuda:0"):
        m._set_readout_map()
    m = _plugin_shell(DenseGGNNChemModel, {"node_mask": _fake_cuda(torch.ones(2, 3), 1)}, {"node_mask": "node_mask"})
    with pytest.raises(GgnnError, match="node_mask must be on cuda:0"):
        m._set_readout_map()
    assert not m.engine.lib.calls


def test_torch_readout_takes_a_tensor_list_without_numpy():
    """ChemModel._graph_nodes_list (the readout at padded hidden sizes) converts a tensor with torch, not through NumPy."""
    import torch
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    m = SparseGGNNChemModel.__new__(SparseGGNNChemModel)
    m.placeholders = {"graph_nodes_list": "graph_nodes_list"}
    m.device = torch.device("cpu")
    t = torch.tensor([0, 0, 2], dtype=torch.int32)
    m.feed = {"graph_nodes_list": t}
    out = m._graph_nodes_list()
    assert out.dtype == torch.long and out.tolist() == [0, 0, 2]
    m.feed = {"graph_nodes_list": _fake_cuda(t)}   # np.asarray of a CUDA tensor raises: this path must not call it
    import unittest.mock as mock
    with mock.patch("gated_graph_neural_network_samples_b200.chem_model.np.asarray", side_effect=AssertionError("np.asarray was called")):
        assert m._graph_nodes_list().tolist() == [0, 0, 2]


# ---------------------------------------------------------------------------------------------------------------- kernel resources
def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def test_map_kernels_have_no_stack_frame_and_no_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump is not available")
    from gated_graph_neural_network_samples_b200 import _build, _lib
    _lib.load()
    out = subprocess.run([exe, "-res-usage", _build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1) if "ro_map" in m.group(1) else None
            continue
        if name is not None and "REG:" in line:
            found[name] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            name = None
    kernels = ("graph_map_kernel", "node_ids_kernel", "dense_map_kernel")
    assert len(found) == len(kernels) and all(any(k in f for f in found) for k in kernels), sorted(found)
    for k, r in found.items():
        print("%s %s" % (k, r))
        assert r["STACK"] == 0 and r.get("LOCAL", 0) == 0, (k, r)
