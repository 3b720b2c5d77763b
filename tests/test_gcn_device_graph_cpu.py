"""CPU-only: the ABI of sparse GCN batches built on the device (``ggnn_set_graph_gcn_device``, DESIGN 2.16) -- the header declaration and
its documented promises, the exported symbol and its ctypes signature, the NULL engine, the Python checks that refuse a bad feed before any
call, the plug-in's route, and the resources of the new kernel (no stack frame, no spills).  Bytes, bits and refusals against the host
builder are in tests/test_gpu_gcn_device_graph.py."""
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


def _block(h):
    """The header's comment block over the entry."""
    end = h.index("int ggnn_set_graph_gcn_device(")
    return h[h.rindex("/*", 0, end):end]


def test_header_declares_the_entry_and_documents_its_promises():
    h = _header()
    assert ("int ggnn_set_graph_gcn_device(ggnn_engine* e, int32_t num_nodes, int64_t nnz, const int64_t* adjacency_list, "
            "ggnn_stream_t stream);") in h
    b = _block(h)
    assert "synchronises `stream` two or three times" in b
    assert "does not depend on the order of any atomic" in b
    assert "No edge is copied to the host" in b
    assert "ggnn_prepare_graph_gcn_message_weighted + ggnn_set_graph_prepared" in b
    for code in ("GGNN_ERANGE", "GGNN_EINVAL", "GGNN_EUNSUPPORTED"):
        assert code in b, code


def test_symbol_is_exported_with_its_signature():
    from gated_graph_neural_network_samples_b200 import _lib
    lib = _lib.load()
    fn = lib.ggnn_set_graph_gcn_device
    assert fn.restype is C.c_int
    assert fn.argtypes == [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]


def test_null_engine_is_refused_without_a_device():
    from gated_graph_neural_network_samples_b200 import _lib
    lib = _lib.load()
    codes = {k: int(v) for k, v in re.findall(r"(GGNN_E[A-Z]+) = (-?\d+)", _header())}
    assert lib.ggnn_set_graph_gcn_device(None, 0, 0, None, None) == codes["GGNN_EINVAL"]
    assert lib.ggnn_set_graph_gcn_device(None, 4, 1, C.c_void_p(16), None) == codes["GGNN_EINVAL"]


class _NoLibrary:
    """Stands in for the library: any call into it fails the test (the feed checks run before the call)."""

    def __getattr__(self, name):
        raise AssertionError("%s was called" % name)


def _bare_engine():
    """A GCNEngine's Python half without a library handle: enough for the feed checks, which run before any call."""
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    eng = GCNEngine.__new__(GCNEngine)
    eng._h = C.c_void_p()
    eng.lib = _NoLibrary()
    eng.D, eng.T, eng.L, eng.device, eng.serial = 32, 1, 2, 0, 0
    return eng


def test_feed_checks_refuse_before_the_call():
    """Type, dtype, shape, contiguity, then device: every bad feed raises GgnnError before the library is touched."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    eng = _bare_engine()
    host = torch.zeros((3, 2), dtype=torch.int64)
    cases = [
        (np.zeros((3, 2), np.int64), "must be a torch tensor"),            # a NumPy array
        ([[0, 1], [1, 0]], "must be a torch tensor"),                       # a Python list
        (host.to(torch.int32), "must be int64"),                            # int32 list
        (host.to(torch.float32), "must be int64"),                          # float list
        (host.to(torch.float64), "must be int64"),
        (host.reshape(-1), "must be [nnz, 2]"),                             # flat
        (host.reshape(1, 3, 2), "must be [nnz, 2]"),                        # 3-d
        (torch.zeros((2, 3), dtype=torch.int64), "must be [nnz, 2]"),       # [2, nnz] (the PyG layout)
        (torch.zeros((3, 4), dtype=torch.int64)[:, :2], "must be contiguous"),
        (torch.zeros((2, 3), dtype=torch.int64).t(), "must be contiguous"),
        (host, "must be on cuda:0"),                                        # a host tensor
    ]
    for lst, text in cases:
        with pytest.raises(GgnnError, match=re.escape(text)):
            eng.set_graph_gcn_device(5, lst)
    with pytest.raises(GgnnError, match=re.escape("num_nodes must be >= 0")):
        eng.set_graph_gcn_device(-1, host)
    assert eng.serial == 0   # no refused call counts as an upload


def test_plugin_routes_cuda_lists_to_the_device_entry():
    """compute_final_node_representations takes set_graph_gcn_device when the feed's adjacency_list is a CUDA tensor, passes the weights
    as the autograd node's trailing input, and keeps set_graph_gcn for host feeds."""
    import inspect
    from gated_graph_neural_network_samples_b200 import chem_gcn
    src = inspect.getsource(chem_gcn.SparseGCNChemModel.compute_final_node_representations)
    assert "set_graph_gcn_device(" in src and "self.engine.set_graph_gcn(h0.shape[0]" in src
    assert "*weights, *aw)" in src
    assert "set_graph_gcn_device" in chem_gcn.propagate.__doc__
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    assert "set_message_weights(w)" in GCNEngine.set_graph_gcn_device.__doc__


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def test_pairs_kernel_has_no_stack_frame_and_no_spills():
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
            name = m.group(1) if "dg_gcn" in m.group(1) else None
            continue
        if name is not None and "REG:" in line:
            found[name] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            name = None
    assert len(found) == 1 and "gcn_pairs_kernel" in next(iter(found)), sorted(found)
    for k, r in found.items():
        print("%s %s" % (k, r))
        assert r["STACK"] == 0 and r.get("LOCAL", 0) == 0, (k, r)
