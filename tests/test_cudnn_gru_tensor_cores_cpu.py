"""CPU: CudnnCompatibleGRUCell at the configured precision (GGNN_CELL_CUDNN_GRU_TENSOR_CORES), everything a host can check.

With ``cell = 3`` on bf16x3 / bf16 every batch takes the streaming wgmma plan, four launches per timestep (gather-GEMM, gate GEMM, the
cell's hidden-projection GEMM, candidate GEMM), five with tensor-core propagation attention.  Checked here without a GPU: the ABI constant
and the keyword; the plan text at every width class from 20 to 512, T = 1 / 4 / 16, both tensor-core precisions, with and without
attention; what must not change (fp32 and GGNN_ATT_FP32 give the cell-2 plan and image bytes, GRU and RNN ignore the keyword); the dense
refusals; the host dataset's batch plans; the plug-ins' option; and the streaming kernel's instances in the built library.
"""
import ctypes as C
import functools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import _lib, engine, packing, synthetic
from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GgnnError, PreparedGraph, make_config
from tests.test_attention_edges_cpu import NUM_SMS, batch
from tests.test_backward_plans_cpu import model

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ggnn_b200.h")
CELL = "CudnnCompatibleGRUCell"
STREAM_CUDNN = (r"^wgmma-%s STREAM\+cudnn-gru\(4 launches per step: gather-GEMM, gate GEMM, hidden-projection GEMM, candidate GEMM\) "
                r"tiles=\d+ DP=%d ")
STREAM_ATT_CUDNN = (r"^wgmma-%s STREAM\+attention\+cudnn-gru\(5 launches per step: attention, gather-GEMM, gate GEMM, hidden-projection "
                    r"GEMM, candidate GEMM\) tiles=\d+ DP=%d ")
WIDTHS = (20, 100, 128, 132, 256, 512)


def cudnn_model(D, attention=False, **kw):
    return model(CELL, D, act="tanh", attention=attention, **kw)


def prep(params, T, adj, indeg, precision="bf16x3", tc=True, save=True, att_tc=False):
    return PreparedGraph.host_only(params, T, adj, indeg, precision=precision, num_sms=NUM_SMS, save_for_backward=save,
                                   attention_tensor_cores=att_tc, cudnn_gru_tensor_cores=tc)


def test_header_enum_and_binding_agree():
    text = open(HEADER).read()
    got = {k: int(v) for k, v in re.findall(r"(GGNN_CELL_[A-Z_0-9]+) = (\d+)", text)}
    assert got == {"GGNN_CELL_GRU": 0, "GGNN_CELL_RNN": 1, "GGNN_CELL_CUDNN_GRU": 2,
                   "GGNN_CELL_CUDNN_GRU_TENSOR_CORES": _lib.CELL_CUDNN_GRU_TENSOR_CORES}
    assert {k: v for k, v in engine.CELL_CODES.items()} == {"gru": 0, "rnn": 1, "cudnncompatiblegrucell": 2}
    p = cudnn_model(8)
    assert make_config(p, 4)[0].cell == 2
    assert make_config(p, 4, cudnn_gru_tensor_cores=True)[0].cell == _lib.CELL_CUDNN_GRU_TENSOR_CORES
    for cell, code in (("GRU", 0), ("RNN", 1)):
        assert make_config(model(cell, 8), 4, cudnn_gru_tensor_cores=True)[0].cell == code


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("kind", ["t1", "hubs", "t16_all"])   # 1, 4 and 16 edge types
def test_plans_stream_at_every_width(kind, precision):
    adj, indeg, T = batch(kind)
    for D in WIDTHS:
        DP = (D + 15) // 16 * 16
        g = prep(cudnn_model(D), T, adj, indeg, precision)
        assert re.search(STREAM_CUDNN % (precision, DP), g.info()["plan"]), (D, g.info()["plan"])
        assert g.info()["streaming"]
        # binary streaming tables: one-message pairs are copies, and there is no vslot (the plan is not all-virtual without attention)
        assert g.stream_tables()["vslot"] is None
        assert (g.arrays(T)["pair_src"] >= 0).any()
        plan = prep(cudnn_model(D, attention=True), T, adj, indeg, precision, att_tc=True).info()["plan"]
        assert re.search(STREAM_ATT_CUDNN % (precision, DP), plan), (D, plan)


def test_value_3_on_fp32_is_value_2():
    """Plan text and image bytes identical, with and without save_for_backward, at a fused and at a per-timestep fp32 width; so with
    GGNN_ATT_FP32 attention at a tensor-core precision."""
    adj, indeg, T = batch("self_dup")
    for D in (36, 260):
        for save in (False, True):
            a, b = prep(cudnn_model(D), T, adj, indeg, "fp32", tc=False, save=save), prep(cudnn_model(D), T, adj, indeg, "fp32", tc=True, save=save)
            assert a.info() == b.info() and "+cudnn-gru" in a.info()["plan"]
            np.testing.assert_array_equal(a.image(), b.image())
            pa = cudnn_model(D, attention=True)
            a, b = prep(pa, T, adj, indeg, "bf16x3", tc=False, save=save), prep(pa, T, adj, indeg, "bf16x3", tc=True, save=save)
            assert a.info() == b.info() and a.info()["plan"].startswith("fp32-"), a.info()["plan"]
            np.testing.assert_array_equal(a.image(), b.image())


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_value_2_stays_on_fp32(precision):
    adj, indeg, T = batch("hubs")
    for D in (36, 260):
        plan = prep(cudnn_model(D), T, adj, indeg, precision, tc=False).info()["plan"]
        assert plan.startswith("fp32-") and "+cudnn-gru" in plan, plan


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("cell", ["GRU", "RNN"])
def test_other_cells_ignore_the_keyword(cell, precision):
    adj, indeg, T = batch("hubs")
    for D in (36, 260):
        for save in (False, True):
            p = model(cell, D, act="tanh")
            a, b = prep(p, T, adj, indeg, precision, tc=False, save=save), prep(p, T, adj, indeg, precision, tc=True, save=save)
            assert a.info() == b.info()
            np.testing.assert_array_equal(a.image(), b.image())


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_dense_prepare_and_dense_dataset_refuse_value_3(precision, monkeypatch):
    from tests.test_dense_device_data_cpu import BONDS, flat_of, molecules, params
    p = dict(params(100), graph_rnn_cell=CELL, graph_rnn_activation="tanh")
    A = np.zeros((2, BONDS, 6, 6), np.float32)
    A[:, 0, 1, 0] = 1.0
    flat = flat_of(molecules()[:20], True)
    # value 2 on the dense entries keeps what it does
    assert "+cudnn-gru" in PreparedGraph.host_only_dense(p, BONDS, A, precision=precision).info()["plan"]
    DeviceDataset.host_only_dense(p, BONDS, flat, precision=precision, for_training=False)
    monkeypatch.setattr(engine, "make_config", functools.partial(make_config, cudnn_gru_tensor_cores=True))
    for call in (lambda: PreparedGraph.host_only_dense(p, BONDS, A, precision=precision),
                 lambda: PreparedGraph.host_only_dense_weighted(p, BONDS, 0.5 * A, precision=precision)):
        with pytest.raises(GgnnError, match="CudnnCompatibleGRUCell exists only in the sparse model"):
            call()
    with pytest.raises(GgnnError, match="CudnnCompatibleGRUCell exists only in the sparse model") as ex:
        DeviceDataset.host_only_dense(p, BONDS, flat, precision=precision, for_training=False)
    assert ex.value.code == -4   # GGNN_EUNSUPPORTED


def test_relu_is_refused():
    """The binding asserts tanh like the reference (sparse:106); the C shape check refuses value 3 with ReLU on its own."""
    with pytest.raises(AssertionError):
        make_config(dict(cudnn_model(8), graph_rnn_activation="ReLU"), 4, cudnn_gru_tensor_cores=True)
    cfg, keep = make_config(cudnn_model(8), 4, precision="bf16x3", cudnn_gru_tensor_cores=True)
    cfg.activation = 1   # GGNN_ACT_RELU
    adj, indeg, T = batch("hubs")
    adjs = [np.ascontiguousarray(np.asarray(a, np.int32).reshape(-1, 2)) for a in adj]
    g = PreparedGraph()
    with pytest.raises(GgnnError, match="CudnnCompatibleGRUCell requires the tanh activation"):
        g._fill(g.lib.ggnn_host_prepare_graph_sparse, indeg.shape[0], T, C.byref(cfg), NUM_SMS, 0, indeg.shape[0],
                (C.c_void_p * T)(*[a.ctypes.data for a in adjs]), (C.c_int32 * T)(*[a.shape[0] for a in adjs]), indeg.ctypes.data)


@pytest.mark.parametrize("D", [36, 256])
@pytest.mark.parametrize("save", [False, True])
def test_host_dataset_batches_plan_like_the_prepared_graph(D, save):
    from tests.test_device_data_cpu import batch_ids, packed_graph, plan_of, sparse_graph_set, tile_starts
    T = 4
    flat = packing.FlatSparseGraphs(sparse_graph_set(), T)
    params = cudnn_model(D)
    ds = DeviceDataset.host_only(params, T, flat, precision="bf16x3", num_sms=NUM_SMS, for_training=save, cudnn_gru_tensor_cores=True)
    for ids in batch_ids(flat.num_graphs, seed=D):
        b = ds.prepare_batch(ids, save_for_backward=save)
        packed = packed_graph(flat, ids, D)
        ref = prep(params, T, packed["adjacency_lists"], packed["num_incoming_edges_per_type"], save=save)
        got, want = b.info(), ref.info()
        assert "STREAM+cudnn-gru(4 launches" in want["plan"]
        assert plan_of(got) == plan_of(want), ids
        assert got["image_bytes"] == want["image_bytes"], ids
        np.testing.assert_array_equal(got["tile_start"], tile_starts(ref, T))


# ---------------------------------------------------------------------------------------------------------------- plug-ins
def test_plugin_passes_the_option_to_the_engine(tmp_path, monkeypatch):
    from gated_graph_neural_network_samples_b200 import chem_sparse
    from tests.test_chem_model_cpu import StandInEngine, StandInPropagation
    seen = []

    class Recording(StandInEngine):
        def __init__(self, params, num_edge_types, device=0, precision="fp32", **kw):
            seen.append(kw)
            super().__init__(params, num_edge_types, device, precision)

    monkeypatch.setattr(chem_sparse, "PropagationEngine", Recording)
    monkeypatch.setattr(chem_sparse, "_propagation_function", lambda: StandInPropagation)
    mols = synthetic.make_molecules(40, seed=1)
    cfg = {"hidden_size": 16, "graph_rnn_cell": CELL, "num_epochs": 1, "batch_size": 200}
    base = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:30], "--valid_data": mols[30:], "--config": cfg}
    a = chem_sparse.SparseGGNNChemModel(dict(base, **{"--precision": "bf16x3", "--cudnn-gru-tensor-cores": True}))
    b = chem_sparse.SparseGGNNChemModel(dict(base, **{"--precision": "bf16x3"}))
    chem_sparse.SparseGGNNChemModel(dict(base, **{"--precision": "bf16x3", "--cudnn-gru-tensor-cores": True, "--attention-tensor-cores": True}))
    assert seen == [{"cudnn_gru_tensor_cores": True}, {}, {"attention_tensor_cores": True, "cudnn_gru_tensor_cores": True}]
    # a command-line option, not a params key: the same params, so checkpoints move between the two
    assert a.params == b.params


def test_dense_and_gcn_plugins_refuse_the_option(tmp_path):
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    mols = synthetic.make_molecules(20, seed=1)
    args = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:15], "--valid_data": mols[15:],
            "--cudnn-gru-tensor-cores": True, "--config": {"hidden_size": 16, "batch_size": 8}}
    for cls in (DenseGGNNChemModel, SparseGCNChemModel):
        with pytest.raises(Exception, match="--cudnn-gru-tensor-cores applies to the sparse GGNN model"):
            cls(args)


# ---------------------------------------------------------------------------------------------------------------- the kernel
def test_stream_instances_have_no_stack_frame():
    """The cell's epilogues are runtime branches of the existing instances: still twelve, none with a stack frame or local memory."""
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    if exe is None:
        pytest.skip("cuobjdump is not available")
    from gated_graph_neural_network_samples_b200 import _build
    _lib.load()
    out = subprocess.run([exe, "-res-usage", _build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            res[name] = {n: int(v) for n, v in re.findall(r"([A-Z_]+):(\d+)", line)}
            name = None
    stream = sorted(n for n in res if "ggnn_stream_kernel" in n)
    assert len(stream) == 12, stream
    assert all(res[n]["STACK"] == 0 and res[n]["LOCAL"] == 0 for n in stream), {n: res[n] for n in stream}
