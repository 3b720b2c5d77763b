"""CPU-only: the ABI of sparse batches built on the device (``ggnn_set_graph_sparse_device``, DESIGN 2.15) -- the header declaration, the
exported symbol and its ctypes signature, the Python checks that refuse a bad feed before any call, and the resources of the builder's
kernels (no stack frame, no spills).  Bytes, bits and refusals against the host builder are in tests/test_gpu_device_graph.py."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 4


def _header():
    with open(os.path.join(ROOT, "include", "ggnn_b200.h")) as f:
        return re.sub(r"\s+", " ", f.read())


def test_header_declares_the_entry_and_documents_its_reads():
    h = _header()
    assert ("int ggnn_set_graph_sparse_device(ggnn_engine* e, int32_t num_nodes, const int32_t* const* adjacency_lists, const int32_t* num_edges, "
            "const float* num_incoming_edges_per_type, int32_t message_weighted, ggnn_stream_t stream);") in h
    assert "synchronises `stream` two or three times" in h
    assert "does not depend on the order of any atomic" in h


def test_symbol_is_exported_with_its_signature():
    from gated_graph_neural_network_samples_b200 import _lib
    lib = _lib.load()
    fn = lib.ggnn_set_graph_sparse_device
    assert fn.restype is C.c_int
    assert fn.argtypes == [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_void_p, C.c_int32, C.c_void_p]


def test_null_engine_is_refused_without_a_device():
    from gated_graph_neural_network_samples_b200 import _lib
    lib = _lib.load()
    codes = {k: int(v) for k, v in re.findall(r"(GGNN_E[A-Z]+) = (-?\d+)", _header())}
    counts = (C.c_int32 * T)(0, 0, 0, 0)
    ptrs = (C.c_void_p * T)()
    assert lib.ggnn_set_graph_sparse_device(None, 0, ptrs, counts, None, 0, None) == codes["GGNN_EINVAL"]


def _bare_engine():
    """A PropagationEngine's Python half without a library handle: enough for the feed checks, which run before any call."""
    from gated_graph_neural_network_samples_b200 import _lib
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine.__new__(PropagationEngine)
    eng._h = C.c_void_p()
    eng.lib = _lib.load()
    eng.T, eng.D, eng.device = T, 32, 0
    return eng


def test_feed_checks_refuse_before_the_call():
    import torch
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    eng = _bare_engine()
    host = [torch.zeros((3, 2), dtype=torch.int32) for _ in range(T)]
    cases = [
        (5, [np.zeros((3, 2), np.int32)] * T, None, "torch tensor on cuda:0"),   # NumPy arrays
        (5, host, None, "torch tensor on cuda:0"),                               # host tensors
        (5, host[:3], None, "expected 4 adjacency lists"),
        (-1, host, None, "num_nodes must be >= 0"),
    ]
    for V, lists, table, text in cases:
        with pytest.raises(GgnnError, match=re.escape(text)):
            eng.set_graph_sparse_device(V, lists, table)


def test_plugin_routes_cuda_lists_to_the_device_entry():
    """compute_final_node_representations takes set_graph_sparse_device when every adjacency list of the feed is a CUDA tensor, and keeps
    set_graph_sparse for host feeds."""
    import inspect
    from gated_graph_neural_network_samples_b200 import chem_sparse
    src = inspect.getsource(chem_sparse.SparseGGNNChemModel.compute_final_node_representations)
    assert "set_graph_sparse_device(" in src and "self.engine.set_graph_sparse(adjacency_lists" in src
    assert "set_graph_sparse_device" in chem_sparse.propagate.__doc__


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


KERNELS = ("count_kernel", "summary_kernel", "cut_flags_kernel", "cut_list_kernel", "indeg_kernel", "denom_kernel", "csr_src_kernel",
           "source_csr_kernel", "virtual_flags_kernel", "stream_rows_kernel", "tile_kernel")


def test_builder_kernels_have_no_stack_frame_and_no_spills():
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
            k = re.match(r"_ZN4ggnn2dg(\d+)(\w+)", m.group(1))
            name = k.group(2)[:int(k.group(1))] if k else None
            continue
        if name is not None and "REG:" in line:
            found[name] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            name = None
    assert sorted(found) == sorted(KERNELS), sorted(found)
    for k, r in found.items():
        assert r["STACK"] == 0 and r.get("LOCAL", 0) == 0, (k, r)
