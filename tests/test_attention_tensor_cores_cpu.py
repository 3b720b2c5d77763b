"""CPU: propagation attention on the tensor-core precisions (GGNN_ATT_TENSOR_CORES), everything a host can check.

With ``use_propagation_attention = 2`` on bf16x3 / bf16, every batch takes the streaming wgmma plan, on which every (target, type) pair
with messages is a virtual row weighted through ``vslot`` by the step's probabilities (a lone message weighs 1 / (1 + 1e-7), not 1).
Checked here without a GPU: the ABI constants; the plan text at every padded width class, T = 1 / 4 / 16, GRU and RNN, both tensor-core
precisions; what must not change (fp32 gives the mode-1 plan and image bytes, CudnnCompatibleGRUCell stays on fp32, 17 edge types and the
dense prepare are refused); the streaming tables against a NumPy restatement from the edge lists, across host thread counts; the host
dataset's batch plans; that a prepared graph rebuilt in place has the bytes of a fresh build (the device dataset's image, assembled from
zeros, must equal it); the plug-in's option; and the new kernel's resources in the built library.
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import _lib, packing, synthetic
from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GgnnError, PreparedGraph
from tests.test_attention_edges_cpu import NUM_SMS, att_model, batch, wire
from tests.test_backward_plans_cpu import component_graph

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ggnn_b200.h")
STREAM_ATT = r"^wgmma-%s STREAM\+attention\(4 launches per step: attention, gather-GEMM, gate GEMM, candidate GEMM\) tiles=\d+ DP=%d "
# one hidden size per padded width class the streaming kernels have (DP 16 .. 128 in steps of 16, then 272, 288, 320, 384, 512)
WIDTHS = (4, 20, 36, 52, 68, 84, 100, 116, 128, 260, 276, 316, 384, 512)


def prep(params, T, adj, indeg, precision="bf16x3", tc=True, save=True, **kw):
    return PreparedGraph.host_only(params, T, adj, indeg, precision=precision, num_sms=NUM_SMS, save_for_backward=save,
                                   attention_tensor_cores=tc, **kw)


def molecules(n=24, T=4, seed=3):
    b = packing.pack_sparse_batch(packing.process_raw_graphs_sparse(synthetic.make_molecules(n, seed=seed, num_bond_types=T)), 8, T)
    return b["adjacency_lists"], np.asarray(b["num_incoming_edges_per_type"], np.float32)


def test_header_enum_and_binding_agree():
    text = open(HEADER).read()
    got = {k: int(v) for k, v in re.findall(r"(GGNN_ATT_[A-Z_0-9]+) = (\d+)", text)}
    assert got == {"GGNN_ATT_OFF": _lib.ATT_OFF, "GGNN_ATT_FP32": _lib.ATT_FP32, "GGNN_ATT_TENSOR_CORES": _lib.ATT_TENSOR_CORES}
    from gated_graph_neural_network_samples_b200.engine import make_config
    p = att_model(8)
    assert make_config(p, 4)[0].use_propagation_attention == _lib.ATT_FP32
    assert make_config(p, 4, attention_tensor_cores=True)[0].use_propagation_attention == _lib.ATT_TENSOR_CORES
    assert make_config(dict(p, use_propagation_attention=False), 4, attention_tensor_cores=True)[0].use_propagation_attention == _lib.ATT_OFF


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("cell", ["GRU", "RNN"])
@pytest.mark.parametrize("kind", ["t1", "hubs", "t16_all"])
def test_mode_2_plans_stream_at_every_width(kind, cell, precision):
    adj, indeg, T = batch(kind)
    for D in WIDTHS:
        DP = (D + 15) // 16 * 16
        plan = prep(att_model(D, cell=cell), T, adj, indeg, precision).info()["plan"]
        assert re.search(STREAM_ATT % (precision, DP), plan), (D, plan)


def test_mode_2_on_fp32_is_mode_1():
    """Plan text and image bytes identical, with and without save_for_backward, at a fused and a per-timestep fp32 width."""
    adj, indeg, T = batch("self_dup")
    for D in (36, 260):
        for save in (False, True):
            a, b = prep(att_model(D), T, adj, indeg, "fp32", tc=False, save=save), prep(att_model(D), T, adj, indeg, "fp32", tc=True, save=save)
            assert a.info() == b.info()
            np.testing.assert_array_equal(a.image(), b.image())


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_cudnn_gru_stays_on_fp32(precision):
    adj, indeg, T = batch("hubs")
    for D in (36, 260):
        plan = prep(att_model(D, cell="CudnnCompatibleGRUCell"), T, adj, indeg, precision).info()["plan"]
        assert plan.startswith("fp32-") and "+attention+cudnn-gru" in plan, plan


def test_seventeen_edge_types_and_the_dense_prepare_are_refused():
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    adj, indeg = component_graph(17, V_target=60, seed=2)
    with pytest.raises(GgnnError, match="propagation attention supports at most 16 edge types"):
        prep(att_model(8), 17, adj, indeg)
    with pytest.raises(GgnnError, match="propagation attention supports at most 16 edge types"):
        PropagationEngine(att_model(8), 17, precision="bf16x3", attention_tensor_cores=True)
    A = np.zeros((2, 4, 6, 6), np.float32)
    A[:, 0, 1, 0] = 1.0
    with pytest.raises(GgnnError, match="propagation attention exists only in the sparse model"):
        PreparedGraph.host_only_dense(att_model(8), 4, A, precision="bf16x3")


# ---------------------------------------------------------------------------------------------------------------- streaming tables
def restated_tables(adj, V, T):
    """From the edge lists alone: the stable target-CSR (messages in type-major list order), then every (target, type) row with messages
    as a virtual row in row order, with its sources, count + first seven sources, first slot, and the first virtual row of every
    128-row tile."""
    src = np.concatenate([np.asarray(a, np.int64).reshape(-1, 2)[:, 0] for a in adj])
    tgt = np.concatenate([np.asarray(a, np.int64).reshape(-1, 2)[:, 1] for a in adj])
    typ = np.concatenate([np.full(np.asarray(a).reshape(-1, 2).shape[0], t) for t, a in enumerate(adj)])
    row = tgt * T + typ
    order = np.argsort(row, kind="stable")
    csr_src = src[order]
    counts = np.bincount(row, minlength=V * T)
    row_ptr = np.concatenate([[0], np.cumsum(counts)])
    rows = np.flatnonzero(counts)
    vptr = np.concatenate([[0], np.cumsum(counts[rows])])
    vinfo = np.zeros((rows.size, 8), np.int64)
    vinfo[:, 0] = counts[rows]
    for i, r in enumerate(rows):
        s = csr_src[row_ptr[r]:row_ptr[r + 1]][:7]
        vinfo[i, 1:1 + s.size] = s
    ntiles = (V + 127) // 128
    tile_vptr = np.searchsorted(rows, np.minimum(np.arange(ntiles + 1) * 128, V) * T)
    pair = np.full(ntiles * 128 * T, -1, np.int64)
    pair[rows] = -(2 + np.arange(rows.size))
    return {"vrow_ptr": vptr, "vsrc": csr_src, "vinfo": vinfo, "vslot": row_ptr[rows], "tile_vptr": tile_vptr, "pair_src": pair}


def big_hub_with_loops_and_duplicates():
    """A target of in-degree 1100 (one source sends it three messages in one type), self-loops beside other messages, a node whose only
    message is a self-loop, and a duplicate pair under two types; 4 edge types."""
    edges = [(s, 0, s % 4) for s in range(1, 1101)] + [(7, 0, 3), (7, 0, 3)]
    edges += [(s, s, s % 4) for s in range(1, 1200, 9)] + [(1201, 1201, 2), (5, 1202, 1), (5, 1202, 1), (6, 1202, 0), (6, 1202, 2)]
    return wire(1203, 4, edges)


GRAPHS = {"molecules": lambda: molecules(60), "big_hub": big_hub_with_loops_and_duplicates,
          "self_dup": lambda: batch("self_dup")[:2], "t16_ends": lambda: batch("t16_ends")[:2]}


@pytest.mark.parametrize("threads", ["1", "2", "3", "8"])
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_every_pair_with_messages_is_a_virtual_row(graph, threads, monkeypatch):
    monkeypatch.setenv("GGNN_HOST_THREADS", threads)
    adj, indeg = GRAPHS[graph]()
    V, T = indeg.shape
    g = prep(att_model(100), T, adj, indeg)
    got, want = g.stream_tables(), restated_tables(adj, V, T)
    assert got["vslot"] is not None
    for k in ("vrow_ptr", "vsrc", "vinfo", "vslot", "tile_vptr"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    np.testing.assert_array_equal(g.arrays(T)["pair_src"], want["pair_src"])
    # the same tables whatever the thread count: the image is one function of the batch
    monkeypatch.setenv("GGNN_HOST_THREADS", "1")
    np.testing.assert_array_equal(g.image(), prep(att_model(100), T, adj, indeg).image())


@pytest.mark.parametrize("tc,precision,D", [(True, "bf16x3", 36), (True, "bf16x3", 260), (False, "bf16x3", 260), (False, "bf16x3", 36),
                                             (False, "fp32", 36)])
def test_an_image_is_one_function_of_its_batch(tc, precision, D):
    """A prepared graph rebuilt in place after a larger batch of another shape has the bytes of a fresh build, alignment gaps and the room
    of empty sections included: the device-assembled dataset image, which starts from zeros, is compared with it byte for byte."""
    params = att_model(D)
    big_adj, big_indeg = big_hub_with_loops_and_duplicates()
    adj, indeg = molecules(24)
    T = indeg.shape[1]
    g = prep(params, T, big_adj, big_indeg, precision, tc=tc)
    fresh = prep(params, T, adj, indeg, precision, tc=tc).image()
    for first in ((big_adj, big_indeg), ([np.zeros((0, 2), np.int32)] * T, np.zeros((0, T), np.float32)), (big_adj, big_indeg)):
        prep(params, T, *first, precision, tc=tc, reuse=g)
        np.testing.assert_array_equal(prep(params, T, adj, indeg, precision, tc=tc, reuse=g).image(), fresh)


def test_binary_streaming_batches_keep_their_tables():
    """Without attention (and with mode 1) a streaming batch keeps its rule: one-message pairs are copies and there is no vslot."""
    adj, indeg = molecules(60)
    V, T = indeg.shape
    p = dict(att_model(256), use_propagation_attention=False)
    a, b = prep(p, T, adj, indeg, tc=False), prep(p, T, adj, indeg, tc=True)
    np.testing.assert_array_equal(a.image(), b.image())
    assert a.stream_tables()["vslot"] is None
    assert (a.arrays(T)["pair_src"] >= 0).any()


@pytest.mark.parametrize("D", [36, 256])
@pytest.mark.parametrize("save", [False, True])
def test_host_dataset_batches_plan_like_the_prepared_graph(D, save):
    from tests.test_device_data_cpu import batch_ids, packed_graph, plan_of, sparse_graph_set, tile_starts
    T = 4
    flat = packing.FlatSparseGraphs(sparse_graph_set(), T)
    params = att_model(D)
    ds = DeviceDataset.host_only(params, T, flat, precision="bf16x3", num_sms=NUM_SMS, for_training=save, attention_tensor_cores=True)
    for ids in batch_ids(flat.num_graphs, seed=D):
        b = ds.prepare_batch(ids, save_for_backward=save)
        packed = packed_graph(flat, ids, D)
        ref = prep(params, T, packed["adjacency_lists"], packed["num_incoming_edges_per_type"], save=save)
        got, want = b.info(), ref.info()
        assert "STREAM+attention" in want["plan"]
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
    cfg = {"hidden_size": 16, "use_propagation_attention": True, "num_epochs": 1, "batch_size": 200}
    base = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:30], "--valid_data": mols[30:], "--config": cfg}
    chem_sparse.SparseGGNNChemModel(dict(base, **{"--precision": "bf16x3", "--attention-tensor-cores": True}))
    chem_sparse.SparseGGNNChemModel(dict(base, **{"--precision": "bf16x3"}))
    assert seen == [{"attention_tensor_cores": True}, {}]


def test_dense_and_gcn_plugins_refuse_the_option(tmp_path):
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    mols = synthetic.make_molecules(20, seed=1)
    args = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:15], "--valid_data": mols[15:],
            "--attention-tensor-cores": True, "--config": {"hidden_size": 16, "batch_size": 8}}
    for cls in (DenseGGNNChemModel, SparseGCNChemModel):
        with pytest.raises(Exception, match="--attention-tensor-cores applies to the sparse GGNN model"):
            cls(args)


# ---------------------------------------------------------------------------------------------------------------- the kernel
def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def test_attention_pre_pass_has_no_stack_frame_and_the_stream_instances_stay():
    exe = _cuobjdump()
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
    pre = [n for n in res if "attention_chunk_kernel" in n]
    assert len(pre) == 1, sorted(res)
    assert res[pre[0]]["STACK"] == 0 and res[pre[0]]["LOCAL"] == 0, res[pre[0]]
    stream = sorted(n for n in res if "ggnn_stream_kernel" in n)
    assert len(stream) == 12, stream   # GATHER x X3 x KS in {1, 2, 4}: the instance set of the streaming plan
    assert all(res[n]["STACK"] == 0 and res[n]["LOCAL"] == 0 for n in stream)
